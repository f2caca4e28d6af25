// xmr_gemm_tf32.cuh -- protected dense matmul on the Hopper tensor cores (BASELINE config 4).
//
// C[M,N] = A[M,K] . B[K,N], fp32 in / fp32 out, row-major, wgmma kind tf32 (operands are read as TF32 = top 19 bits of each
// fp32; fp32 accumulate in registers).  It is the tensor-core realisation of matrix_multiply()
// (tests/matrixMultiply/matrixMultiply.c:95-112, tests/mm_common/mm_common_tmr.c:3-20); the bit-exact integer flavour of
// those loops is xmr_mm.cuh / xmr_mm_tc.cuh.
//
// Redundancy costs FLOPs, not bandwidth:
//   * ONE copy of each A/B tile is staged in shared memory by TMA (128B swizzle, K-major), an mbarrier ring;
//   * every consumer warpgroup issues each wgmma NC times, once per replica, into NC DIFFERENT register accumulators -- the
//     replicas of cloneInsns (cloning.cpp:2189-2204) are NC independent accumulator tiles fed from the same operand bytes;
//   * the epilogue votes the NC accumulators element-wise in registers with the reference's select voter and `fcmp oeq`
//     (synchronization.cpp:57-62,512-522), counts disagreements (:1391-1431), and writes ONE voted C tile.
// Unit = one C element (the `mm_t` store, mm_common_tmr.c:16); local unit index = i*N + j.
// Fault site 0 = the replica's final accumulator value (32 bits) as read for the vote.
//
// TF32 wgmma reads both operands K-major, so B goes through a transposing pre-pass (xmr_gemm_bt) into library scratch first;
// a caller who holds B^T (COAST_MM_B_TRANSPOSED) skips it: the same kernels read the caller's B^T rows in place.
// The same body runs BF16 operands (xmr_gemm_bf16*, operand type Bf16 below): bfloat16 A and B, fp32 accumulators and C,
// wgmma m64n128k16.  16-bit wgmma can read B MN-major, which is what a row-major K x N matrix is, so B is loaded in place from
// the caller's buffer: no pre-pass and no scratch.  A BF16 B^T (COAST_MM_B_TRANSPOSED) is read in place K-major (Bf16T, the
// xmr_gemm_bf16*_bt_* kernels).
// And FP8 operands (xmr_gemm_fp8*, operand type Fp8): E4M3 A and B, fp32 C, wgmma m64n128k32.  The 8-bit wgmma has no transpose
// immediates, so B is read K-major only: as for TF32, a byte-transposing pre-pass (xmr_gemm_bt_u8) writes B^T into scratch, and
// a caller's B^T (COAST_MM_B_TRANSPOSED) is read in place by the same kernels.
// And INT8 operands (xmr_gemm_i8*, operand type I8): s8 A and B laid out as FP8's, wgmma m64n128k32 into s32 accumulators that
// wrap, so C = A . B mod 2^32 exactly; the epilogue votes the int32 words with integer equality.
// And FP16 operands (xmr_gemm_f16*, operand types F16 and F16T): IEEE binary16 A and B in BF16's layout (B in place MN-major, or
// the caller's B^T K-major), wgmma m64n128k16 f16 x f16 into fp32 accumulators.
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, 64 rows of the 128-row tile each.
// Persistent CTAs, one per SM.  Tiles: 128 x 256 unprotected (N % 256 == 0), 128 x 128 otherwise; the accumulators of a
// replica are 64 x 128 wgmma fragments (64 fp32 registers per thread), so TMR holds 192 accumulator registers per thread.
//
// CTA pairs (xmr_gemm_tf32p_*, cluster 2 x 1 x 1): two CTAs compute the two 128-row halves of a 256 x BN tile and share its
// B tile: each CTA loads half of it with a TMA multicast into both CTAs' shared memory, halving the L2 -> SM traffic for B.
// Every element sees the same wgmma sequence as in the single-CTA kernel, so the outputs are bit-identical.
#pragma once
#include "xmr_common.cuh"
#include "xmr_mm_grp.cuh"

namespace xmr {
namespace gemm {

constexpr int BM = XMR_WG_BM;
constexpr uint32_t ROW_BYTES = 128;                  // a k-block of either operand type is one 128-byte swizzle row of A
constexpr int WG_N = 128;                            // wgmma N per instruction
constexpr uint32_t A_STAGE = BM * ROW_BYTES;         // 16 KiB
constexpr int CTA_THREADS = XMR_WG_THREADS;          // warpgroup 0 = producer, 1-2 = consumers
template <int NC, bool WIDE = (NC == 1)> struct Geom {         // WIDE: 128 x 256 tiles (unprotected, N % 256 == 0)
    static constexpr int BN = (int)xmr_gemm_bn(WIDE);
    static constexpr int NSUB = BN / WG_N;
    static constexpr int STAGES = (int)xmr_gemm_stages(WIDE);   // 192 KiB of operand stages either way
    static constexpr uint32_t B_STAGE = BN * ROW_BYTES;          // TF32: [BN rows of B^T][128 B]; BF16: [BN / 64 boxes][64 k-rows][128 B]
    // 1 KiB alignment slack, the stages, then full[] and empty[]
    static_assert(1023u + STAGES * (A_STAGE + B_STAGE) + 2u * STAGES * sizeof(uint64_t) <= xmr_gemm_smem(WIDE),
                  "stages and barriers fit the launch's shared memory");
};
constexpr uint32_t GROUP_M_DEFAULT = 16;             // tile rasterisation: 16 tile-rows per group, column-major inside
constexpr uint32_t GROUP_M = GROUP_M_DEFAULT;        // (xmr_mm_tc.cuh uses the fixed value)

// Persistent CTAs take tiles blockIdx.x, +grid, ...; consecutive tile ids therefore run concurrently.  Row-major ids would make
// one wave touch a few A row-blocks and ALL of B; grouping 16 tile-rows and walking columns inside the group keeps a wave on
// ~16 A row-blocks x ~9 B column-blocks, which the 50 MB L2 holds.
__device__ __forceinline__ void tile_coords(uint32_t tile, uint32_t tiles_m, uint32_t tiles_n, uint32_t group_m, uint32_t& tm, uint32_t& tn) {
    const uint32_t per_group = group_m * tiles_n;
    const uint32_t g = tile / per_group, w = tile - g * per_group;
    const uint32_t rows = min(group_m, tiles_m - g * group_m);
    tm = g * group_m + w % rows;
    tn = w / rows;
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// L2 eviction-priority hints (xmr_args.mode bit 8): A loads evict_last (the row block is reused by every column tile of its
// group), B loads and C stores evict_first.
__device__ __forceinline__ uint64_t l2_policy_evict_last() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t l2_policy_evict_first() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t l2_policy_normal() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(pol) : "memory");
}
// the box lands at the same shared-memory offset in every CTA of `mask` and completes its bytes on each one's barrier at `bar`'s offset
__device__ __forceinline__ void tma_load_2d_mcast(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint16_t mask, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5, %6;"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_v2_hint(void* p, uint32_t x, uint32_t y, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.b32 [%0], {%1, %2}, %3;" ::"l"(p), "r"(x), "r"(y), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_b32_hint(void* p, uint32_t x, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(p), "r"(x), "l"(pol) : "memory");
}
// two fp32 values (bit patterns) rounded to bfloat16, to nearest even, into one bf16x2: lo in bits [0,16), hi in [16,32)
__device__ __forceinline__ uint32_t pack_bf16x2_rn(uint32_t lo, uint32_t hi) {
    uint32_t d;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "r"(hi), "r"(lo));
    return d;
}
// the same into one f16x2 (IEEE binary16): finite values of 65520 or more in magnitude become infinities
__device__ __forceinline__ uint32_t pack_f16x2_rn(uint32_t lo, uint32_t hi) {
    uint32_t d;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "r"(hi), "r"(lo));
    return d;
}
// an f16 (the low 16 bits of h) as the fp32 of the same value, exactly
__device__ __forceinline__ float f16_widen(uint32_t h) {
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"((unsigned short)h));
    return f;
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the barrier at this shared-memory offset in CTA `rank` of the cluster (this CTA included)
__device__ __forceinline__ void mbar_arrive_rank(uint64_t* bar, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(r) : "memory");
}
// mbarrier wait that cannot hang the GPU: a protocol error (a lost arrival) traps after ~2^26 polls instead of spinning
__device__ __forceinline__ void mbar_wait_or_trap(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    for (uint32_t spins = 0; spins < (1u << 26); ++spins) {
        uint32_t done;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return;
    }
    asm volatile("trap;");
}

// ---- wgmma (sm_90a) -------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major operand in the 128-byte swizzle (TMA CU_TENSOR_MAP_SWIZZLE_128B): start >> 4
// [0,14), LBO [16,30) (unused for this layout, 1), SBO = 1024 B between 8-row groups [32,46), layout SWIZZLE_128B (1) [62,64).
// A step of 32 bytes along K inside the 128-byte row is an add of 2 to the start field.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma boundary
template <class T, int R> __device__ __forceinline__ void wg_fence_regs(T (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(*reinterpret_cast<uint32_t*>(&d[i])) :: "memory");
}
template <int NEW> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(NEW)); }
template <int NEW> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(NEW)); }

// D (+)= A . B^T with both operands K-major in shared memory; fragment layout of D (64 x N, one warpgroup): thread t holds
// d[4j + 2h + e] = D[16 (t / 32) + (t % 32) / 4 + 8h][8j + 2 (t % 4) + e]
__device__ __forceinline__ void wgmma_tf32_m64n128k8(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db));
}

// Shared-memory matrix descriptor of an MN-major 16-bit operand in the 128-byte swizzle: what TMA (CU_TENSOR_MAP_SWIZZLE_128B)
// leaves of a row-major K x N matrix loaded in boxes of 64 columns x 64 k-rows.  A box is 64 k-rows of 128 bytes (64 columns),
// 8 KiB; the 16-byte chunks of a row are XORed with (k-row % 8), which is the swizzle atom of 64 columns x 8 k-rows = 1 KiB.
// start >> 4 [0,14); LBO [16,30) = 8192 B from one 64-column box to the next; SBO [32,46) = 1024 B from one group of 8 k-rows
// to the next; layout SWIZZLE_128B (1) [62,64).  One k16 step (two 8-row groups) is 2048 bytes further into the box: an add
// of 128 to the start field; the next 128 columns are two boxes on: an add of 1024.
__device__ __forceinline__ uint64_t wg_desc_mn(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// D (+)= A . B with A K-major and B MN-major (the transpose immediates 0, 1) in shared memory, or, TRANS_B = 0, D (+)= A . B^T
// with both operands K-major (0, 0); D's fragment layout as above
template <int TRANS_B = 1>
__device__ __forceinline__ void wgmma_bf16_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, %66;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "n"(TRANS_B));
}
// the same with IEEE binary16 operands
template <int TRANS_B = 1>
__device__ __forceinline__ void wgmma_f16_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, %66;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "n"(TRANS_B));
}

// D (+)= A . B^T with both operands K-major, E4M3 x E4M3 (the 8-bit wgmma takes no transpose immediates); D's fragment layout as above
__device__ __forceinline__ void wgmma_e4m3_m64n128k32(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db));
}

// D (+)= A . B^T with both operands K-major, s8 x s8 into s32 accumulators (no .satfinite: the sums wrap mod 2^32); D's fragment
// layout as above
__device__ __forceinline__ void wgmma_s8_m64n128k32(int32_t (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db));
}

// The operand types of gemm_body.  Both stage 128-byte k-blocks (BK elements) and step A's descriptor by 32 bytes (WG_K elements)
// per wgmma; they differ in the instruction and in how B reaches shared memory:
//   Tf32: B^T rows from the transposing pre-pass, K-major like A; TMA boxes of B_BOX rows of B^T at 128 bytes per row;
//   Bf16: B in place, MN-major; TMA boxes of 64 columns x BK k-rows (128 bytes is the widest box row this swizzle takes), 8 KiB
//         each, so column c of the tile lies in the box at byte 128 c -- the same place B^T row c has for Tf32.
//   Bf16T: the caller's B^T (COAST_MM_B_TRANSPOSED: N rows of K) read in place, K-major like A and like Tf32's B^T: the same
//         boxes of B_BOX rows of 128 bytes (64 k), a k16 step is 32 bytes, and the wgmma's B transpose immediate is 0.
struct Tf32 {
    using Acc = float;
    static constexpr int BK = XMR_GEMM_BK, WG_K = 8;
    static constexpr bool B_IN_PLACE = false;
    static constexpr uint32_t B_KSTEP = 32 >> 4;                 // descriptor start field per wgmma k step
    static constexpr __host__ __device__ int b_box(bool pair) { return (int)xmr_gemm_b_box(pair); }
    static __device__ __forceinline__ uint64_t desc_b(uint32_t saddr) { return wg_desc(saddr); }
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) { wgmma_tf32_m64n128k8(d, da, db); }
};
struct Bf16 {
    using Acc = float;
    static constexpr int BK = XMR_GEMM_BF16_BK, WG_K = 16;
    static constexpr bool B_IN_PLACE = true;
    static constexpr uint32_t B_KSTEP = (WG_K * ROW_BYTES) >> 4;
    static constexpr __host__ __device__ int b_box(bool) { return (int)XMR_GEMM_BF16_B_BOX; }
    static __device__ __forceinline__ uint64_t desc_b(uint32_t saddr) { return wg_desc_mn(saddr); }
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) { wgmma_bf16_m64n128k16(d, da, db); }
};
struct Bf16T {
    using Acc = float;
    static constexpr int BK = XMR_GEMM_BF16_BK, WG_K = 16;
    static constexpr bool B_IN_PLACE = false;
    static constexpr uint32_t B_KSTEP = 32 >> 4;
    static constexpr __host__ __device__ int b_box(bool pair) { return (int)xmr_gemm_b_box(pair); }
    static __device__ __forceinline__ uint64_t desc_b(uint32_t saddr) { return wg_desc(saddr); }
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) { wgmma_bf16_m64n128k16<0>(d, da, db); }
};
//   F16, F16T: IEEE binary16 operands in Bf16's and Bf16T's layouts; only the wgmma's operand type differs.
struct F16 : Bf16 {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) { wgmma_f16_m64n128k16(d, da, db); }
};
struct F16T : Bf16T {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) { wgmma_f16_m64n128k16<0>(d, da, db); }
};
//   Fp8: E4M3 operands, B^T K-major like Tf32's (the pre-pass's scratch or the caller's B^T): a k-block is 128 elements, the same
//        128-byte row, and a k32 step is 32 bytes, the same descriptor step as Tf32's.  The accumulator is the wgmma's own
//        (DESIGN.md §6: for FP8 it is narrower than fp32), as with torch._scaled_mm(use_fast_accum=True).
struct Fp8 {
    using Acc = float;
    static constexpr int BK = XMR_GEMM_FP8_BK, WG_K = 32;
    static constexpr bool B_IN_PLACE = false;
    static constexpr uint32_t B_KSTEP = 32 >> 4;
    static constexpr __host__ __device__ int b_box(bool pair) { return (int)xmr_gemm_b_box(pair); }
    static __device__ __forceinline__ uint64_t desc_b(uint32_t saddr) { return wg_desc(saddr); }
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) { wgmma_e4m3_m64n128k32(d, da, db); }
};
//   I8: s8 operands, laid out as Fp8's (the same k-blocks, descriptors, pre-pass and B^T boxes), into s32 accumulators that wrap:
//       C = sum_k a_ik b_kj mod 2^32, exact for any K.  The epilogue votes them as integers (see epilogue).
struct I8 {
    using Acc = int32_t;
    static constexpr int BK = XMR_GEMM_FP8_BK, WG_K = 32;
    static constexpr bool B_IN_PLACE = false;
    static constexpr uint32_t B_KSTEP = 32 >> 4;
    static constexpr __host__ __device__ int b_box(bool pair) { return (int)xmr_gemm_b_box(pair); }
    static __device__ __forceinline__ uint64_t desc_b(uint32_t saddr) { return wg_desc(saddr); }
    static __device__ __forceinline__ void mma(int32_t (&d)[64], uint64_t da, uint64_t db) { wgmma_s8_m64n128k32(d, da, db); }
};

__device__ __forceinline__ void wgmma_u8_m64n32k32(uint32_t (&d)[16], uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.u8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
        : "l"(da), "l"(db));
}

__device__ __forceinline__ void wgmma_u8_m64n64k32(uint32_t (&d)[32], uint64_t da, uint64_t db) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.u8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(da), "l"(db));
}

template <class X, class Y> struct Same { static constexpr bool value = false; };
template <class X> struct Same<X, X> { static constexpr bool value = true; };
// C's element type (the OUT parameter of the epilogue and gemm_body): fp32 (I8: its s32 words), bfloat16 or f16
enum COut : int { C_F32 = 0, C_BF16 = 1, C_F16 = 2 };
template <int OUT> struct CElem { using T = uint16_t; };
template <> struct CElem<C_F32> { using T = float; };
__device__ __forceinline__ uint32_t acc_word(float x) { return __float_as_uint(x); }     // an accumulator's 32-bit word
__device__ __forceinline__ uint32_t acc_word(int32_t x) { return (uint32_t)x; }
// Epilogue of one consumer thread: vote the NC accumulators of its fragment element by element with the reference's select
// voter / `fcmp oeq`, count, ONE store of the voted value.  Columns [n0 + 128 sub, ...) for sub < nsub_t.
// GROUPED: C starts at row ro[0] (c_grp) and rows from row_end on belong to the next product: no vote, tally, flip or store.
// SCALED (xmr_scaled_fp8*): each replica's value, after the fault hook, becomes (acc x sa) x sb, two fp32 multiplies rounded to
// nearest, and the vote is on those.  sa: the A scale of row `row` is sa[row] (ROWWISE) or sa[0]; sb: the B scale of column
// `col` is sb[col] or sb[0] (the caller offsets both to the tile's product).  The two layouts are two instances, so neither
// carries the other's loads and branches next to the accumulators.  Every replica reads the one copy
// of a scale (-noMemReplication's load rule), after the main loop, so nothing of it is live next to the accumulators.
// OUT C_BF16 (xmr_o16_*, COAST_MM_OUT_BF16; not with SCALED): C holds bfloat16.  Each replica rounds its thread's two values
// (after the fault hook) into one bf16x2 with cvt.rn, the vote and the tally run on the 16-bit halves (`fcmp oeq` on the widened
// values, the majority voter bitwise on the pair), and one 4-byte store writes the voted pair: its own branch, with its own pair vote.
// OUT C_F16 (xmr_h16_*, COAST_MM_OUT_F16) is the same branch with cvt.rn.f16x2.f32 and cvt.f32.f16 for the widening.
// Integer accumulators (AccT int32_t, xmr_gemm_i8*; neither SCALED nor 16-bit C): the vote is integer equality (`icmp eq`) on the
// two's-complement words, with the select or the bitwise majority voter.  The fp32 vote would be wrong on them: `fcmp oeq` takes a
// bit-31 flip of a zero C (0x80000000, -0.0) as equal to +0.0, and every C whose pattern is a NaN as a disagreement.  It shares
// the fp32 branch -- word read, fault hook, vote and tally -- but for the compare; C is written with the same 8-byte pair stores.
// The fault hook and the word reads stay written out in each branch: as inline helpers shared by the branches (over arrays,
// over scalar references, with the vote or without), they changed the SASS of the TMR kernels (DESIGN.md §5.2).
template <int NC, int NSUB, bool INJECT, bool GROUPED = false, bool SCALED = false, bool ROWWISE = false, int OUT = C_F32,
          class AccT = float>
__device__ __forceinline__ void epilogue(const xmr_args& a, Tally& tally, AccT (&acc)[NC][NSUB][64], uint32_t row0, uint32_t n0, uint32_t nsub_t,
                                         bool hints, uint64_t pol_c, typename CElem<OUT>::T* c_grp = nullptr, uint32_t row_end = 0,
                                         const float* sa = nullptr, const float* sb = nullptr) {
    static_assert(!(SCALED && OUT != C_F32), "scaled GEMM_FP8 has no 16-bit-output epilogue");
    constexpr bool INT_ACC = !Same<AccT, float>::value;
    static_assert(!INT_ACC || (Same<AccT, int32_t>::value && !SCALED && OUT == C_F32), "integer accumulators: s32, unscaled, 4-byte C");
    using CT = typename CElem<OUT>::T;
    const uint32_t flags = a.flags;
    const bool majority = flags & COAST_F_MAJORITY_VOTER;
    CT* C = GROUPED ? c_grp : static_cast<CT*>(a.out);
    const uint32_t lane = threadIdx.x & 31;
    constexpr bool rowwise = SCALED && ROWWISE;
    float s_row[2] = {1.f, 1.f}, s_col = 1.f;
    if constexpr (SCALED) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {                       // a masked row of a grouped tile loads nothing
            const uint32_t row = row0 + 8 * h;
            if (!GROUPED || row < row_end) s_row[h] = __ldg(sa + (rowwise ? row : 0u));
        }
        if (!rowwise) s_col = __ldg(sb);
    }
#pragma unroll
    for (int sub = 0; sub < NSUB; ++sub) {
        if ((uint32_t)sub >= nsub_t) break;
#pragma unroll
        for (int j = 0; j < WG_N / 8; ++j) {
            float2 s_pair = make_float2(s_col, s_col);       // the B scales of this thread's two columns (an even first column)
            if constexpr (SCALED) {
                if constexpr (rowwise) s_pair = __ldg(reinterpret_cast<const float2*>(sb + n0 + sub * WG_N + 8 * j + 2 * (lane & 3)));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t row = row0 + 8 * h, col = n0 + sub * WG_N + 8 * j + 2 * (lane & 3);
                if constexpr (GROUPED) { if (row >= row_end) continue; }
                const unsigned long long local0 = (unsigned long long)row * a.N + col;
                if constexpr (OUT != C_F32) {
                    uint32_t x[3][2];                            // [replica][element]: the accumulators after the fault hook
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = 4 * j + 2 * h + e;
                        x[0][e] = __float_as_uint(acc[0][sub][i]);
                        x[1][e] = NC > 1 ? __float_as_uint(acc[NC > 1 ? 1 : 0][sub][i]) : x[0][e];
                        x[2][e] = NC > 2 ? __float_as_uint(acc[NC > 2 ? 2 : 0][sub][i]) : x[0][e];
                        if (INJECT) {
                            Fault f = fault_for_unit(a, NC, local0 + e, [](uint32_t) { return 32u; });
                            if (f.active) {
                                tally.injected++;
                                const uint32_t mk = 1u << f.bit;
                                if (f.replica == 0) x[0][e] ^= mk; else if (f.replica == 1) x[1][e] ^= mk; else x[2][e] ^= mk;
                            }
                        }
                    }
                    uint32_t p0, p1, p2;                                           // every replica rounds its own pair
                    if constexpr (OUT == C_F16) {
                        p0 = pack_f16x2_rn(x[0][0], x[0][1]);
                        p1 = NC > 1 ? pack_f16x2_rn(x[1][0], x[1][1]) : p0;
                        p2 = NC > 2 ? pack_f16x2_rn(x[2][0], x[2][1]) : p0;
                    } else {
                        p0 = pack_bf16x2_rn(x[0][0], x[0][1]);
                        p1 = NC > 1 ? pack_bf16x2_rn(x[1][0], x[1][1]) : p0;
                        p2 = NC > 2 ? pack_bf16x2_rn(x[2][0], x[2][1]) : p0;
                    }
                    uint32_t o = p0;
                    if (NC == 3 && majority) o = (p0 & p1) | (p0 & p2) | (p1 & p2);
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const uint32_t half = e ? 0xFFFF0000u : 0x0000FFFFu;       // element e's bfloat16 / f16
                        float f0, f1, f2;
                        if constexpr (OUT == C_F16) {
                            f0 = f16_widen(e ? p0 >> 16 : p0); f1 = f16_widen(e ? p1 >> 16 : p1); f2 = f16_widen(e ? p2 >> 16 : p2);
                        } else {
                            f0 = __uint_as_float(e ? p0 & half : p0 << 16); f1 = __uint_as_float(e ? p1 & half : p1 << 16);
                            f2 = __uint_as_float(e ? p2 & half : p2 << 16);
                        }
                        uint32_t bad = 0;
                        if (NC == 2) bad = (f0 == f1) ? 0u : 1u;
                        if (NC == 3) {
                            const bool c01 = (f0 == f1), c02 = (f0 == f2);       // fcmp oeq on the widened values
                            if (!majority && !c01) o = (o & ~half) | (p2 & half);
                            bad = (c01 && c02) ? 0u : 1u;
                        }
                        tally.unit_exit<NC>(bad, 1u, flags, a.unit_base + local0 + e);
                    }
                    CT* dst = C + local0;
                    if (hints) st_b32_hint(dst, o, pol_c);
                    else *reinterpret_cast<uint32_t*>(dst) = o;
                } else {
                    uint32_t o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = 4 * j + 2 * h + e;
                        uint32_t r0 = acc_word(acc[0][sub][i]);
                        uint32_t r1 = NC > 1 ? acc_word(acc[NC > 1 ? 1 : 0][sub][i]) : r0;
                        uint32_t r2 = NC > 2 ? acc_word(acc[NC > 2 ? 2 : 0][sub][i]) : r0;
                        if (INJECT) {
                            Fault f = fault_for_unit(a, NC, local0 + e, [](uint32_t) { return 32u; });
                            if (f.active) {
                                tally.injected++;
                                uint32_t mk = 1u << f.bit;
                                if (f.replica == 0) r0 ^= mk; else if (f.replica == 1) r1 ^= mk; else r2 ^= mk;
                            }
                        }
                        if constexpr (SCALED) {                      // every replica scales its own value; explicit _rn: no contraction
                            const float sr = s_row[h], sc = e ? s_pair.y : s_pair.x;
                            r0 = __float_as_uint(__fmul_rn(__fmul_rn(__uint_as_float(r0), sr), sc));
                            if (NC > 1) r1 = __float_as_uint(__fmul_rn(__fmul_rn(__uint_as_float(r1), sr), sc));
                            if (NC > 2) r2 = __float_as_uint(__fmul_rn(__fmul_rn(__uint_as_float(r2), sr), sc));
                        }
                        const float f0 = __uint_as_float(r0), f1 = __uint_as_float(r1), f2 = __uint_as_float(r2);
                        uint32_t vote = r0, bad = 0;
                        if (NC == 2) bad = (INT_ACC ? r0 == r1 : f0 == f1) ? 0u : 1u;
                        if (NC == 3) {
                            const bool c01 = INT_ACC ? r0 == r1 : f0 == f1, c02 = INT_ACC ? r0 == r2 : f0 == f2;   // icmp eq / fcmp oeq
                            vote = majority ? ((r0 & r1) | (r0 & r2) | (r1 & r2)) : (c01 ? r0 : r2);
                            bad = (c01 && c02) ? 0u : 1u;
                        }
                        o[e] = vote;
                        tally.unit_exit<NC>(bad, 1u, flags, a.unit_base + local0 + e);
                    }
                    CT* dst = C + local0;
                    if (hints) st_v2_hint(dst, o[0], o[1], pol_c);
                    else *reinterpret_cast<uint2*>(dst) = make_uint2(o[0], o[1]);
                }
            }
        }
    }
}

// PAIR: the CTA pair of a cluster 2 x 1 x 1 computes a 256 x BN tile, rank r the rows [128 r, 128 r + 128); each rank loads half
// of the tile's B^T rows and multicasts them to both, so a stage is released only when the consumers of BOTH CTAs are done with it.
// GROUPED (single CTAs with 128 x 128 tiles, xmr_mm_grp.cuh): a.M products of their own row counts, `ro` their row offsets and
// `grp` the group block: the tiles come from its tile_start table, A through its rebased map, B^T rows from g N (Bf16: B rows from g K).
// SCALED (xmr_scaled_fp8*): sa and sb are the caller's scales (see epilogue); a row-wise B scale vector holds N entries per product.
// OUT (xmr_o16_*, xmr_h16_*): C holds bfloat16 or f16 at the same element offsets (see epilogue).
template <class OP, int NC, bool INJECT, bool WIDE, bool PAIR, bool GROUPED = false, bool SCALED = false, int OUT = C_F32>
__device__ __forceinline__ void gemm_body(const xmr_args& a, const CUtensorMap* map_a, const CUtensorMap* map_b,
                                          const unsigned long long* ro = nullptr, const uint8_t* grp = nullptr,
                                          const float* sa = nullptr, const float* sb = nullptr) {
    static_assert(!(GROUPED && (PAIR || WIDE)), "grouped launches run on single CTAs with 128 x 128 tiles");
    using G = Geom<NC, WIDE>;
    constexpr int BN = G::BN, NSUB = G::NSUB, STAGES = G::STAGES;
    constexpr uint32_t B_STAGE = G::B_STAGE;
    constexpr int BK = OP::BK, WG_K = OP::WG_K;
    constexpr int B_BOX = OP::b_box(PAIR);                      // B^T rows (Bf16: B columns) per TMA box
    constexpr uint32_t CTAS = PAIR ? 2u : 1u;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023u) & ~(uintptr_t)1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_STAGE;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * (A_STAGE + B_STAGE));
    uint64_t* full = bars;                 // [STAGES]  TMA -> consumers
    uint64_t* empty = bars + STAGES;       // [STAGES]  consumers (of both CTAs of a pair) -> producer(s)

    const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
    const uint32_t worker = blockIdx.x / CTAS, n_workers = gridDim.x / CTAS;
    const uint32_t TM = BM * CTAS;                              // rows of a (pair) tile
    // a batch stacks its products' rows (n_units / N of them, a.M per product); the host keeps every tile inside one product
    const uint32_t tiles_n = a.N / BN, tiles_m = (uint32_t)(a.n_units / a.N) / TM, kblocks = a.K / BK;
    // grouped: R = n_units / N rows from row ro[0] of d_in / d_out, a.M products
    const uint32_t R = GROUPED ? (uint32_t)(a.n_units / a.N) : 0u, n_grp = GROUPED ? a.M : 0u;
    const uint32_t* ts = GROUPED ? reinterpret_cast<const uint32_t*>(grp + XMR_MM_GRP_TILES) : nullptr;
    const unsigned long long ro0 = GROUPED ? __ldg(ro) : 0ull;
    const uint32_t n_tiles = GROUPED ? __ldg(ts + n_grp) * tiles_n : tiles_m * tiles_n;
    if constexpr (GROUPED) map_a = reinterpret_cast<const CUtensorMap*>(grp);
    const uint32_t gm1 = (a.mode & XMR_MODE_GROUP_M_MASK) ? (a.mode & XMR_MODE_GROUP_M_MASK) : GROUP_M_DEFAULT;
    const uint32_t group_m = PAIR ? (gm1 > 1u ? gm1 / 2u : 1u) : gm1;   // pair tiles are 256 rows: half as many tile-rows per group
    const bool hints = (a.mode & XMR_MODE_L2_HINTS) != 0;
    // Wave quantisation (WIDE only): e.g. 512 tiles on 132 CTAs are 3.9 rounds.  When the last, partial round holds at most half
    // the workers, each of its tiles is split into two 128-column halves, so the tail costs half a round: virtual tile ids
    // [0, sched_full) are whole tiles, [sched_full, n_virtual) are halves (two consecutive ids per tile).
    uint32_t sched_full = n_tiles, n_virtual = n_tiles;
    if (WIDE) {
        const uint32_t whole = (n_tiles / n_workers) * n_workers, rem = n_tiles - whole;
        if (rem && 2u * rem <= n_workers && !(a.mode & XMR_MODE_NO_TAIL_SPLIT)) { sched_full = whole; n_virtual = whole + 2u * rem; }
    }
    auto decode = [&](uint32_t v, uint32_t& tm, uint32_t& n_off, uint32_t& bn_t) {
        uint32_t w = v, h = 0, tn;
        bn_t = BN;
        if (v >= sched_full) { w = sched_full + ((v - sched_full) >> 1); h = (v - sched_full) & 1u; bn_t = BN / 2; }
        tile_coords(w, tiles_m, tiles_n, group_m, tm, tn);
        n_off = tn * BN + h * (BN / 2);
    };

    if (threadIdx.x == 0) {
        // the rebased A map was written by the pre-pass through the generic proxy
        if constexpr (GROUPED) asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(map_a) : "memory");
        tma_prefetch_desc(map_a); tma_prefetch_desc(map_b);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2u * CTAS); }   // 2 consumer warpgroups per CTA
        fence_barrier_init();
    }
    __syncthreads();
    if (PAIR) cluster_sync_all();                               // the peer's barriers exist before anything signals them

    const int wg = threadIdx.x >> 7;
    if (wg == 0) {
        // ===== producer warpgroup: one thread issues every TMA
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {
            uint32_t it = 0;
            const uint64_t pol_a = hints ? l2_policy_evict_last() : l2_policy_normal(), pol_b = hints ? l2_policy_evict_first() : l2_policy_normal();
            for (uint32_t tile = worker; tile < n_virtual; tile += n_workers) {
                uint32_t tm, n_off, bn_t;
                int m0;
                uint32_t nb;
                if constexpr (GROUPED) {
                    // rows past the product read the next product's rows (masked in the epilogue), or zeros past R
                    const grp::Tile x = grp::tile_of(ro, ro0, R, ts, n_grp, tiles_n, group_m, tile);
                    m0 = (int)(x.start + x.tm * TM); nb = x.g * (OP::B_IN_PLACE ? a.K : a.N); n_off = x.tn * BN; bn_t = BN;
                } else {
                    decode(tile, tm, n_off, bn_t);
                    m0 = (int)(tm * TM + rank * BM);
                    nb = (tm * TM) / a.M * a.N;                     // first B^T row of the tile's product (stacked B^T)
                    if constexpr (OP::B_IN_PLACE) nb = (tm * TM) / a.M * a.K;   // first row of the product's B (stacked B)
                }
                const uint32_t rows_b = bn_t / CTAS;                // B^T rows (Bf16: B columns) this CTA loads (for both CTAs of a pair)
                for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
                    const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                    mbar_wait_or_trap(&empty[s], ph ^ 1u);
                    mbar_arrive_expect_tx(&full[s], A_STAGE + bn_t * ROW_BYTES);
                    tma_load_2d_hint(sA + s * A_STAGE, map_a, &full[s], (int)(kb * BK), m0, pol_a);          // box {BK k, 128 m}
                    for (uint32_t c = 0; c < rows_b / B_BOX; ++c) {
                        const uint32_t r = rank * rows_b + c * B_BOX;                                        // row of the tile's B^T (Bf16: column of its B)
                        const int c0 = OP::B_IN_PLACE ? (int)(n_off + r) : (int)(kb * BK), c1 = OP::B_IN_PLACE ? (int)(nb + kb * BK) : (int)(nb + n_off + r);
                        if (PAIR) tma_load_2d_mcast(sB + s * B_STAGE + r * ROW_BYTES, map_b, &full[s], c0, c1, (uint16_t)3, pol_b);
                        else tma_load_2d_hint(sB + s * B_STAGE + r * ROW_BYTES, map_b, &full[s], c0, c1, pol_b);
                    }
                }
            }
        }
    } else {
        // ===== consumer warpgroups: NC wgmmas per operand pair, one accumulator set per replica, vote in registers
        setmaxnreg_inc<232>();
        const uint32_t t = threadIdx.x & 127;
        const uint32_t a_off = (uint32_t)(wg - 1) * 64u * 128u;      // this warpgroup's 64 rows of the A tile
        const uint64_t pol_c = l2_policy_evict_first();
        Tally tally(a);
        typename OP::Acc acc[NC][NSUB][64];                 // fp32, or s32 for I8
        uint32_t it = 0;
        for (uint32_t tile = worker; tile < n_virtual; tile += n_workers) {
            uint32_t tm, n0, bn_t;
            if constexpr (GROUPED) bn_t = BN;                   // grouped: the tile's place is found after the main loop
            else decode(tile, tm, n0, bn_t);
            const uint32_t nsub_t = bn_t / WG_N;
#pragma unroll
            for (int r = 0; r < NC; ++r)
#pragma unroll
                for (int sub = 0; sub < NSUB; ++sub)
#pragma unroll
                    for (int i = 0; i < 64; ++i) acc[r][sub][i] = typename OP::Acc(0);
#pragma unroll
            for (int r = 0; r < NC; ++r)
#pragma unroll
                for (int sub = 0; sub < NSUB; ++sub) wg_fence_regs(acc[r][sub]);
            for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
                const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                mbar_wait_or_trap(&full[s], ph);
                const uint64_t da0 = wg_desc(smem_u32(sA + s * A_STAGE) + a_off), db0 = OP::desc_b(smem_u32(sB + s * B_STAGE));
                wg_fence();
#pragma unroll
                for (int k = 0; k < BK / WG_K; ++k) {
#pragma unroll
                    for (int sub = 0; sub < NSUB; ++sub) {
                        if ((uint32_t)sub >= nsub_t) break;
                        const uint64_t da = da0 + (uint64_t)(2 * k), db = db0 + (uint64_t)(OP::B_KSTEP * k + sub * (WG_N * ROW_BYTES >> 4));
#pragma unroll
                        for (int r = 0; r < NC; ++r) {
                            // with several replica accumulators in flight, ptxas may move one between the asynchronous wgmmas
                            // (seen on the DWC kernel: wrong results); retiring each replica's wgmma before the next keeps them apart
                            if (NC > 1 && r > 0) { wg_commit(); wg_wait<0>(); wg_fence(); }
                            OP::mma(acc[r][sub], da, db);
                        }
                    }
                }
                wg_commit();
                // Retire this stage's wgmmas before anything else runs: no accumulator register may be in flight where the
                // compiler is free to move it (across the loop back-edge), and the stage can be released at once.
                wg_wait<0>();
#pragma unroll
                for (int r = 0; r < NC; ++r)
#pragma unroll
                    for (int sub = 0; sub < NSUB; ++sub) wg_fence_regs(acc[r][sub]);
                if (t == 0) for (uint32_t c = 0; c < CTAS; ++c) mbar_arrive_rank(&empty[s], c);
            }
            // the tile's first row and column for this thread, C's first row (grouped: ro[0], which also indexes the row-wise A
            // scales), the rows it may write and its product (which places its row-wise B scales)
            uint32_t row0, n_t, row_end = 0, prod = 0;
            unsigned long long c_row = 0;
            if constexpr (GROUPED) {
                // found here rather than before the main loop: nothing of it stays live next to the accumulators
                const unsigned long long r0 = __ldg(ro);
                const grp::Tile x = grp::tile_of(ro, r0, R, ts, n_grp, tiles_n, group_m, tile);
                row0 = x.start + x.tm * TM + (uint32_t)(wg - 1) * 64u + 16u * (t >> 5) + ((t & 31) >> 2);
                n_t = x.tn * BN;
                c_row = r0;
                row_end = x.end;
                prod = x.g;
            } else {
                row0 = tm * TM + rank * BM + (uint32_t)(wg - 1) * 64u + 16u * (t >> 5) + ((t & 31) >> 2);
                n_t = n0;
            }
            using CT = typename CElem<OUT>::T;
            CT* const c_grp = GROUPED ? static_cast<CT*>(a.out) + c_row * a.N : nullptr;
            // the two scale layouts are two instances: one epilogue that chose at run time spilled (DESIGN.md §10 item 11).  The
            // row-wise offsets are computed in the row-wise call only.
            if (SCALED && (a.mode & XMR_MODE_SCALE_ROWWISE))
                epilogue<NC, NSUB, INJECT, GROUPED, SCALED, true, OUT>(a, tally, acc, row0, n_t, nsub_t, hints, pol_c, c_grp, row_end,
                                                                            sa + c_row,
                                                                            sb + (unsigned long long)(GROUPED ? prod : (tm * TM) / a.M) * a.N);
            else
                epilogue<NC, NSUB, INJECT, GROUPED, SCALED, false, OUT>(a, tally, acc, row0, n_t, nsub_t, hints, pol_c, c_grp, row_end,
                                                                             sa, sb);
        }
        tally.flush(a.counters);
    }
    if (PAIR) cluster_sync_all();                               // nobody leaves while the peer's multicasts / remote arrivals are in flight
}

}  // namespace gemm
}  // namespace xmr

// B (batch x K x N, row-major) -> B^T (batch x N x K, one stacked (batch N) x K operand): the K-major operand TF32 wgmma reads.
// 32 x 32 tiles through shared memory.
extern "C" __global__ void __launch_bounds__(XMR_PREPASS_THREADS)
xmr_gemm_bt(const float* __restrict__ B, float* __restrict__ Bt, unsigned int K, unsigned int N, unsigned int batch) {
    __shared__ float tile[32][33];
    const unsigned int tiles_n = N / 32u, tiles_k = K / 32u;
    const unsigned long long per = (unsigned long long)tiles_n * tiles_k, n_tiles = per * batch;
    for (unsigned long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const unsigned long long b = t / per;
        const unsigned int w = (unsigned int)(t - b * per), k0 = (w / tiles_n) * 32u, n0 = (w % tiles_n) * 32u;
        const float* Bb = B + b * K * N;
        float* Btb = Bt + b * N * K;
        for (int i = threadIdx.x; i < 1024; i += 256) tile[i >> 5][i & 31] = __ldg(Bb + (size_t)(k0 + (i >> 5)) * N + n0 + (i & 31));
        __syncthreads();
        for (int i = threadIdx.x; i < 1024; i += 256) Btb[(size_t)(n0 + (i >> 5)) * K + k0 + (i & 31)] = tile[i & 31][i >> 5];
        __syncthreads();
    }
}

// B (batch x K x N bytes, row-major) -> B^T ((batch N) x K bytes): xmr_gemm_bt for 1-byte elements (GEMM_FP8).  64 x 64-byte
// tiles through shared memory; each thread moves 4-byte words both ways and packs four bytes of a column into one word.
extern "C" __global__ void __launch_bounds__(XMR_PREPASS_THREADS)
xmr_gemm_bt_u8(const uint8_t* __restrict__ B, uint8_t* __restrict__ Bt, unsigned int K, unsigned int N, unsigned int batch) {
    __shared__ uint32_t tile[64][17];                    // [k][n / 4]: a 68-byte row keeps a column's bytes on different banks
    const uint8_t* t8 = reinterpret_cast<const uint8_t*>(tile);
    const unsigned int tiles_n = N / 64u, tiles_k = K / 64u;
    const unsigned long long per = (unsigned long long)tiles_n * tiles_k, n_tiles = per * batch;
    for (unsigned long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const unsigned long long b = t / per;
        const unsigned int w = (unsigned int)(t - b * per), k0 = (w / tiles_n) * 64u, n0 = (w % tiles_n) * 64u;
        const uint8_t* Bb = B + b * K * N;
        uint8_t* Btb = Bt + b * N * K;
        for (int i = threadIdx.x; i < 1024; i += XMR_PREPASS_THREADS)
            tile[i >> 4][i & 15] = __ldg(reinterpret_cast<const uint32_t*>(Bb + (size_t)(k0 + (i >> 4)) * N + n0) + (i & 15));
        __syncthreads();
        for (int i = threadIdx.x; i < 1024; i += XMR_PREPASS_THREADS) {
            const int n = i >> 4, k = 4 * (i & 15);
            const uint32_t v = (uint32_t)t8[k * 68 + n] | (uint32_t)t8[(k + 1) * 68 + n] << 8 | (uint32_t)t8[(k + 2) * 68 + n] << 16 |
                               (uint32_t)t8[(k + 3) * 68 + n] << 24;
            reinterpret_cast<uint32_t*>(Btb + (size_t)(n0 + n) * K + k0)[i & 15] = v;
        }
        __syncthreads();
    }
}

// ---- the entry points -------------------------------------------------------------------------------------------
// XMR_GEMM_FAMILY(OP, SCALED, OUT, STEM, BT, ORDER, GN1, XP, XA) declares one family's 20 kernels on gemm_body<OP, ...>,
// at inj 0 and 1 each (<i>):
//   STEM BT <nc>            NC 1-3: 128 x 256 tiles at NC 1 (unprotected, N % 256 == 0), 128 x 128 at NC 2-3
//   STEM n BT <nc1>         NC 1: 128 x 128 tiles (N a multiple of 128 but not of 256)
//   STEM p BT <nc>          NC 1-3: CTA pairs (cluster 2 x 1 x 1), 256 x 256 (unprotected) / 256 x 128 pair tiles
//   STEM GN1 BT _grp_inj<i>_nc1, STEM BT _grp_inj<i>_nc<2,3>
//                           grouped (COAST_MM_GROUPED): single CTAs, 128 x 128 tiles; after the maps they take `ro`, the
//                           caller's row offsets, and `grp`, the group block the pre-pass wrote (xmr_mm_grp.cuh)
// <nc> is _inj<i>_nc<n> (ORDER IN) or, for TF32's kernels that came before the grouped ones, _nc<n>_inj<i> (ORDER NI).  BT is
// _bt for BF16's B^T kernels, GN1 is the n that the grouped NC 1 kernels of TF32 and BF16 carry.  XP and XA are the extra
// parameters after the maps (grouped: after ro and grp) and their arguments to gemm_body, each list opening with its comma:
// () or, scaled, (, const float* sa, const float* sb) and (, sa, sb).  For example, FP8 is xmr_gemm_fp8_inj<i>_nc<1,2,3>,
// xmr_gemm_fp8n_inj<i>_nc1, xmr_gemm_fp8p_inj<i>_nc<1,2,3> and xmr_gemm_fp8_grp_inj<i>_nc<1,2,3>; TF32 is
// xmr_gemm_tf32{,p}_nc<1,2,3>_inj<i>, xmr_gemm_tf32n_nc1_inj<i>, xmr_gemm_tf32n_grp_inj<i>_nc1 and xmr_gemm_tf32_grp_inj<i>_nc<2,3>.
#define XMR_LIST(...) __VA_ARGS__
#define XMR_GEMM_NAME_IN(STEM, V, BT, NC, INJ) STEM##V##BT##_inj##INJ##_nc##NC
#define XMR_GEMM_NAME_NI(STEM, V, BT, NC, INJ) STEM##V##BT##_nc##NC##_inj##INJ
#define XMR_GEMM_NAME_GRP(STEM, V, BT, NC, INJ) STEM##V##BT##_grp_inj##INJ##_nc##NC
#define XMR_NO_CLUSTER
#define XMR_PAIR_CLUSTER __cluster_dims__(2, 1, 1)
#define XMR_GEMM_ENTRY(NAME, CLUSTER, OP, NC, INJ, WIDE, PAIR, GROUPED, SCALED, OUT, PARAMS, ARGS)                         \
    extern "C" __global__ void CLUSTER __launch_bounds__(xmr::gemm::CTA_THREADS, 1)                                        \
    NAME(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap map_a,                                    \
         const __grid_constant__ CUtensorMap map_b XMR_LIST PARAMS) {                                                      \
        xmr::gemm::gemm_body<xmr::gemm::OP, NC, INJ != 0, WIDE, PAIR, GROUPED, SCALED, xmr::gemm::OUT>(a, &map_a, &map_b XMR_LIST ARGS); \
    }
#define XMR_GEMM_ONE(V, NC, INJ, WIDE, PAIR, CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                            \
    XMR_GEMM_ENTRY(XMR_GEMM_NAME_##ORDER(STEM, V, BT, NC, INJ), CLUSTER, OP, NC, INJ, WIDE, PAIR, false, SCALED, OUT,      \
                   XP, (, nullptr, nullptr XMR_LIST XA))
#define XMR_GEMM_GRP(V, NC, INJ, OP, SCALED, OUT, STEM, BT, XP, XA)                                                        \
    XMR_GEMM_ENTRY(XMR_GEMM_NAME_GRP(STEM, V, BT, NC, INJ), XMR_NO_CLUSTER, OP, NC, INJ, false, false, true, SCALED, OUT,  \
                   (, const unsigned long long* ro, const uint8_t* grp XMR_LIST XP), (, ro, grp XMR_LIST XA))
#define XMR_GEMM_FAMILY(OP, SCALED, OUT, STEM, BT, ORDER, GN1, XP, XA)                                                     \
    XMR_GEMM_ONE(, 1, 0, true, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                            \
    XMR_GEMM_ONE(, 2, 0, false, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                           \
    XMR_GEMM_ONE(, 3, 0, false, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                           \
    XMR_GEMM_ONE(, 1, 1, true, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                            \
    XMR_GEMM_ONE(, 2, 1, false, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                           \
    XMR_GEMM_ONE(, 3, 1, false, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                           \
    XMR_GEMM_ONE(n, 1, 0, false, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                          \
    XMR_GEMM_ONE(n, 1, 1, false, false, XMR_NO_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                          \
    XMR_GEMM_ONE(p, 1, 0, true, true, XMR_PAIR_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                          \
    XMR_GEMM_ONE(p, 2, 0, false, true, XMR_PAIR_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                         \
    XMR_GEMM_ONE(p, 3, 0, false, true, XMR_PAIR_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                         \
    XMR_GEMM_ONE(p, 1, 1, true, true, XMR_PAIR_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                          \
    XMR_GEMM_ONE(p, 2, 1, false, true, XMR_PAIR_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                         \
    XMR_GEMM_ONE(p, 3, 1, false, true, XMR_PAIR_CLUSTER, OP, SCALED, OUT, STEM, BT, ORDER, XP, XA)                         \
    XMR_GEMM_GRP(GN1, 1, 0, OP, SCALED, OUT, STEM, BT, XP, XA)                                                             \
    XMR_GEMM_GRP(, 2, 0, OP, SCALED, OUT, STEM, BT, XP, XA)                                                                \
    XMR_GEMM_GRP(, 3, 0, OP, SCALED, OUT, STEM, BT, XP, XA)                                                                \
    XMR_GEMM_GRP(GN1, 1, 1, OP, SCALED, OUT, STEM, BT, XP, XA)                                                             \
    XMR_GEMM_GRP(, 2, 1, OP, SCALED, OUT, STEM, BT, XP, XA)                                                                \
    XMR_GEMM_GRP(, 3, 1, OP, SCALED, OUT, STEM, BT, XP, XA)

// fp32 C: TF32 (B^T from the transposing pre-pass or the caller), BF16 with B read in place and with B^T read in place, FP8
// (E4M3; B^T from the byte pre-pass or the caller), INT8 (s8, s32 C, integer vote; FP8's layout), FP16 (BF16's layout)
XMR_GEMM_FAMILY(Tf32, false, C_F32, xmr_gemm_tf32, , NI, n, (), ())
XMR_GEMM_FAMILY(Bf16, false, C_F32, xmr_gemm_bf16, , IN, n, (), ())
XMR_GEMM_FAMILY(Bf16T, false, C_F32, xmr_gemm_bf16, _bt, IN, n, (), ())
XMR_GEMM_FAMILY(Fp8, false, C_F32, xmr_gemm_fp8, , IN, , (), ())
XMR_GEMM_FAMILY(I8, false, C_F32, xmr_gemm_i8, , IN, , (), ())
XMR_GEMM_FAMILY(F16, false, C_F32, xmr_gemm_f16, , IN, n, (), ())
XMR_GEMM_FAMILY(F16T, false, C_F32, xmr_gemm_f16, _bt, IN, n, (), ())
// Scaled FP8 (COAST_MM_SCALE_TENSOR / COAST_MM_SCALE_ROWWISE): the scale pointers follow the maps (grouped: ro and grp); every
// replica multiplies its accumulator by the A and B scales before the vote
XMR_GEMM_FAMILY(Fp8, true, C_F32, xmr_scaled_fp8, , IN, , (, const float* sa, const float* sb), (, sa, sb))
// BF16 output (COAST_MM_OUT_BF16): every GEMM_BF16 and GEMM_FP8 kernel once more, named xmr_o16_ + the name without its
// xmr_gemm_ prefix; C holds bfloat16, each replica rounds its values before the vote (see epilogue).  Scaled GEMM_FP8 has no
// BF16-output set: its TMR and DWC kernels spilled 104-296 bytes with it (DESIGN.md §10 item 12)
XMR_GEMM_FAMILY(Bf16, false, C_BF16, xmr_o16_bf16, , IN, n, (), ())
XMR_GEMM_FAMILY(Bf16T, false, C_BF16, xmr_o16_bf16, _bt, IN, n, (), ())
XMR_GEMM_FAMILY(Fp8, false, C_BF16, xmr_o16_fp8, , IN, , (), ())
// FP16 output (COAST_MM_OUT_F16, GEMM_F16 only): every GEMM_F16 kernel once more, named xmr_h16_ + the name without its
// xmr_gemm_ prefix; C holds f16, each replica rounds its values before the vote
XMR_GEMM_FAMILY(F16, false, C_F16, xmr_h16_f16, , IN, n, (), ())
XMR_GEMM_FAMILY(F16T, false, C_F16, xmr_h16_f16, _bt, IN, n, (), ())
