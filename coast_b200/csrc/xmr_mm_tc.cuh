// xmr_mm_tc.cuh -- protected EXACT integer matmul on the tensor cores (wgmma u8 x u8 -> s32).
//
// matrix_multiply() of the reference (tests/mm_common/mm_common_tmr.c:3-20, tests/matrixMultiply/matrixMultiply.c:95-112)
// is integer arithmetic modulo 2^32.  Split every u32 into four u8 limbs, a = sum_i a_i 2^(8i), b = sum_j b_j 2^(8j):
//     a*b mod 2^32 = sum_{i+j<=3} (a_i * b_j) << 8(i+j)
// so C = S0 + (S1 << 8) + (S2 << 16) + (S3 << 24) mod 2^32 with S_d = sum_{i+j=d} A_i . B_j  -- ten u8 x u8 GEMMs whose
// s32 accumulators WRAP (no .satfinite), which keeps every S_d exact modulo 2^32 for any K.  Bit-exact with the reference's
// own loops, at tensor-core rate.
//
// Data path:  xmr_mm_split_a / xmr_mm_split_bt (pre-pass, library scratch): A -> 4 u8 planes [l][M][K], B -> 4 TRANSPOSED
// u8 planes [l][N][K] (both K-major, as integer wgmma requires); TMA (one 3-D box per operand per stage: {128 k, rows, 4 planes})
// -> 2-stage ring; each consumer warpgroup issues, per 32-byte k-step, the 10 limb-pair wgmmas NC times into NC x 4 register
// accumulators (S0..S3 per replica, BN columns each); the epilogue recombines each replica's C from its four accumulators,
// votes element-wise (one mm_t vote per unit), counts, and stores ONE C tile.  Fault site s (`sum` after k-step s) is applied
// lazily and exactly as in xmr_mm_tiled.cuh.  Warp roles as in xmr_gemm_tf32.cuh: warpgroup 0 produces, 1-2 consume.
#pragma once
#include "xmr_common.cuh"
#include "xmr_gemm_tf32.cuh"   // TMA / wgmma helpers (xmr::gemm::*)

namespace xmr {
namespace mmtc {

using namespace xmr::gemm;

constexpr int TBM = XMR_WG_BM, TBK = XMR_MMTC_BK;    // 128 u8 of K = one 128-byte swizzle row = 4 wgmmas of K = 32
// register accumulators per consumer thread: NC x 4 x BN / 2 (TMR: 3 x 4 x 16 = 192)
template <int NC> struct Geom {
    static constexpr int BN = (int)xmr_mmtc_bn(NC);
    static constexpr uint32_t A_STAGE_B = 4u * TBM * TBK;            // 64 KiB: [plane][row][128 B]
    static constexpr uint32_t B_STAGE_B = 4u * BN * TBK;             // 32 / 16 KiB
    static constexpr int STAGES_ = (int)XMR_MMTC_STAGES;
    // 1 KiB alignment slack, the stages, then full[] and empty[]
    static_assert(1023u + STAGES_ * (A_STAGE_B + B_STAGE_B) + 2u * STAGES_ * sizeof(uint64_t) <= xmr_mmtc_smem(NC),
                  "stages and barriers fit the launch's shared memory");
};
template <int BN> __device__ __forceinline__ void wgmma_u8(uint32_t (&d)[BN / 2], uint64_t da, uint64_t db);
template <> __device__ __forceinline__ void wgmma_u8<32>(uint32_t (&d)[16], uint64_t da, uint64_t db) { wgmma_u8_m64n32k32(d, da, db); }
template <> __device__ __forceinline__ void wgmma_u8<64>(uint32_t (&d)[32], uint64_t da, uint64_t db) { wgmma_u8_m64n64k32(d, da, db); }

// GROUPED (xmr_mm_grp.cuh): a.M products of their own row counts; the A planes hold the R rows from ro[0] (xmr_mm_grp_split_a),
// the B^T planes the G products' B; tiles come from the group block's tile_start and rows past a product are masked.
// BT (COAST_MM_B_TRANSPOSED): aux holds B^T, so the planes come from xmr_mm_split_a and only the fault recompute, which reads the
// u32 operands, differs: it reads B^T[col][k].
template <int NC, bool INJECT, bool GROUPED = false, bool BT = false>
__device__ __forceinline__ void body(const xmr_args& a, const CUtensorMap* map_a, const CUtensorMap* map_b,
                                     const unsigned long long* ro = nullptr, const uint8_t* grp = nullptr) {
    using G = Geom<NC>;
    constexpr int BN = G::BN, STAGES_ = G::STAGES_, R = BN / 2;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023u) & ~(uintptr_t)1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES_ * G::A_STAGE_B;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES_ * (G::A_STAGE_B + G::B_STAGE_B));
    uint64_t* full = bars;
    uint64_t* empty = bars + STAGES_;

    // a batch stacks its products' rows (n_units / N of them, a.M per product; no tile straddles two products)
    const uint32_t tiles_n = a.N / BN, tiles_m = (uint32_t)(a.n_units / a.N) / TBM, kblocks = a.K / TBK;
    const uint32_t n_rows = GROUPED ? (uint32_t)(a.n_units / a.N) : 0u, n_grp = GROUPED ? a.M : 0u;
    const uint32_t* ts = GROUPED ? reinterpret_cast<const uint32_t*>(grp + XMR_MM_GRP_TILES) : nullptr;
    const unsigned long long ro0 = GROUPED ? __ldg(ro) : 0ull;
    const uint32_t n_tiles = GROUPED ? __ldg(ts + n_grp) * tiles_n : tiles_m * tiles_n;
    // tile order: GROUP_M tile-rows per group, column-major inside (same L2 argument as the TF32 kernel)
    auto coords = [&](uint32_t tile, uint32_t& tm, uint32_t& tn) { tile_coords(tile, tiles_m, tiles_n, GROUP_M, tm, tn); };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(map_a); tma_prefetch_desc(map_b);
        for (int s = 0; s < STAGES_; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    const int wg = threadIdx.x >> 7;
    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {
            uint32_t it = 0;
            for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                uint32_t tm, tn, m0, nb;
                if constexpr (GROUPED) {
                    const grp::Tile x = grp::tile_of(ro, ro0, n_rows, ts, n_grp, tiles_n, GROUP_M, tile);
                    tn = x.tn; m0 = x.start + x.tm * TBM; nb = x.g * a.N;
                } else {
                    coords(tile, tm, tn);
                    m0 = tm * TBM;
                    nb = (tm * TBM) / a.M * a.N;                // first B^T row of the tile's product (stacked B^T planes)
                }
                for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
                    const uint32_t s = it % STAGES_, ph = (it / STAGES_) & 1u;
                    mbar_wait_or_trap(&empty[s], ph ^ 1u);
                    mbar_arrive_expect_tx(&full[s], G::A_STAGE_B + G::B_STAGE_B);
                    tma_load_3d(sA + s * G::A_STAGE_B, map_a, &full[s], (int)(kb * TBK), (int)m0, 0);               // box {128 k, 128 m, 4 planes}
                    tma_load_3d(sB + s * G::B_STAGE_B, map_b, &full[s], (int)(kb * TBK), (int)(nb + tn * BN), 0);  // box {128 k, BN n, 4 planes}
                }
            }
        }
    } else {
        setmaxnreg_inc<232>();
        const uint32_t t = threadIdx.x & 127, lane = t & 31;
        const uint32_t a_off = (uint32_t)(wg - 1) * 64u * 128u;
        const uint32_t flags = a.flags;
        const bool majority = flags & COAST_F_MAJORITY_VOTER;
        uint32_t* C = static_cast<uint32_t*>(a.out) + (GROUPED ? ro0 * a.N : 0ull);          // grouped: from row ro[0]
        const uint32_t* __restrict__ A32 = static_cast<const uint32_t*>(a.in) + (GROUPED ? ro0 * a.K : 0ull);
        const uint32_t* __restrict__ B32 = static_cast<const uint32_t*>(a.aux);
        Tally tally(a);
        uint32_t acc[NC][4][R];
        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            uint32_t tm, tn;
            if constexpr (GROUPED) tm = tn = 0;                 // grouped: found after the main loop, next to the accumulators
            else coords(tile, tm, tn);
#pragma unroll
            for (int r = 0; r < NC; ++r)
#pragma unroll
                for (int d = 0; d < 4; ++d)
#pragma unroll
                    for (int i = 0; i < R; ++i) acc[r][d][i] = 0u;
#pragma unroll
            for (int r = 0; r < NC; ++r)
#pragma unroll
                for (int d = 0; d < 4; ++d) wg_fence_regs(acc[r][d]);
            for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
                const uint32_t s = it % STAGES_, ph = (it / STAGES_) & 1u;
                mbar_wait_or_trap(&full[s], ph);
                // descriptors differ only in the 14-bit start-address field: base + (plane offset + k*32) >> 4
                const uint64_t da0 = wg_desc(smem_u32(sA + s * G::A_STAGE_B) + a_off), db0 = wg_desc(smem_u32(sB + s * G::B_STAGE_B));
                wg_fence();
#pragma unroll
                for (int k = 0; k < TBK / 32; ++k) {
#pragma unroll
                    for (int d = 0; d < 4; ++d) {            // diagonal d = i + j: shift 8d, accumulator S_d
#pragma unroll
                        for (int i = 0; i <= d; ++i) {
                            const int j = d - i;
                            const uint64_t da = da0 + (uint64_t)((i * (TBM * TBK) + k * 32) >> 4);
                            const uint64_t db = db0 + (uint64_t)((j * (BN * TBK) + k * 32) >> 4);
#pragma unroll
                            for (int r = 0; r < NC; ++r) wgmma_u8<BN>(acc[r][d], da, db);
                        }
                    }
                }
                wg_commit();
                wg_wait<0>();                                   // as in xmr_gemm_tf32.cuh: nothing stays in flight across the back-edge
#pragma unroll
                for (int r = 0; r < NC; ++r)
#pragma unroll
                    for (int d = 0; d < 4; ++d) wg_fence_regs(acc[r][d]);
                if (t == 0) mbar_arrive(&empty[s]);
            }
            uint32_t row_start = 0, row_end = 0, g = 0;
            if constexpr (GROUPED) {
                const grp::Tile x = grp::tile_of(ro, ro0, n_rows, ts, n_grp, tiles_n, GROUP_M, tile);
                tm = x.tm; tn = x.tn; row_start = x.start; row_end = x.end; g = x.g;
            }
            const uint32_t row_base = row_start + tm * TBM + (uint32_t)(wg - 1) * 64u + 16u * (t >> 5) + (lane >> 2);
#pragma unroll
            for (int jj = 0; jj < BN / 8; ++jj) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t row = row_base + 8u * h, col = tn * BN + 8u * jj + 2u * (lane & 3u);
                    if constexpr (GROUPED) { if (row >= row_end) continue; }          // the next product's row: not ours
                    const unsigned long long local0 = (unsigned long long)row * a.N + col;
                    uint32_t o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int q = 4 * jj + 2 * h + e;
                        uint32_t cr[3];
#pragma unroll
                        for (int r = 0; r < NC; ++r) cr[r] = acc[r][0][q] + (acc[r][1][q] << 8) + (acc[r][2][q] << 16) + (acc[r][3][q] << 24);   // mod 2^32
                        uint32_t r0 = cr[0], r1 = NC > 1 ? cr[NC > 1 ? 1 : 0] : r0, r2 = NC > 2 ? cr[NC > 2 ? 2 : 0] : r0;
                        if (INJECT) {
                            Fault f = fault_for_unit(a, NC, local0 + e, [](uint32_t) { return 32u; });
                            if (f.active) {
                                tally.injected++;
                                uint32_t part = 0;          // S_s = partial sum over k <= site, from the original u32 operands
                                const uint32_t* Bp = B32 + (size_t)(GROUPED ? g : row / a.M) * a.K * a.N;    // the element's own product's B
                                for (uint32_t k = 0; k <= f.site; ++k)
                                    part += __ldg(A32 + (size_t)row * a.K + k) * __ldg(BT ? Bp + (size_t)(col + e) * a.K + k : Bp + (size_t)k * a.N + col + e);
                                const uint32_t mk = 1u << f.bit, delta = (part & mk) ? (0u - mk) : mk;
                                if (f.replica == 0) r0 += delta; else if (f.replica == 1) r1 += delta; else r2 += delta;
                            }
                        }
                        uint32_t vote = r0, bad = 0;
                        if (NC == 2) bad = r0 != r1;
                        if (NC == 3) {
                            const bool c01 = r0 == r1, c02 = r0 == r2;
                            vote = majority ? ((r0 & r1) | (r0 & r2) | (r1 & r2)) : (c01 ? r0 : r2);
                            bad = (c01 && c02) ? 0u : 1u;
                        }
                        o[e] = vote;
                        tally.unit_exit<NC>(bad, 1u, flags, a.unit_base + local0 + e);
                    }
                    *reinterpret_cast<uint2*>(C + local0) = make_uint2(o[0], o[1]);
                }
            }
        }
        tally.flush(a.counters);
    }
}

}  // namespace mmtc
}  // namespace xmr

// ---- limb-split pre-pass ---------------------------------------------------------------------------------------
// A (u32, rows x K, row-major) -> planes[l][row][k] (u8).  One thread = 4 consecutive k of one row.
__device__ __forceinline__ void split_a_body(const uint32_t* __restrict__ A, uint8_t* __restrict__ planes, unsigned long long rows,
                                             unsigned long long K) {
    const unsigned long long quads = rows * K / 4ull, stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long q = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += stride) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(A) + q);
        const uint32_t lo = __byte_perm(v.x, v.y, 0x5140u);        // x.b0 y.b0 x.b1 y.b1  (interleave low halves)
        const uint32_t hi = __byte_perm(v.x, v.y, 0x7362u);        // x.b2 y.b2 x.b3 y.b3
        const uint32_t lo2 = __byte_perm(v.z, v.w, 0x5140u), hi2 = __byte_perm(v.z, v.w, 0x7362u);
        uint32_t* p = reinterpret_cast<uint32_t*>(planes);
        const unsigned long long plane = rows * K / 4ull;
        p[q] = __byte_perm(lo, lo2, 0x5410u);                      // plane 0: b0 of x,y,z,w
        p[plane + q] = __byte_perm(lo, lo2, 0x7632u);              // plane 1
        p[2ull * plane + q] = __byte_perm(hi, hi2, 0x5410u);       // plane 2
        p[3ull * plane + q] = __byte_perm(hi, hi2, 0x7632u);       // plane 3
    }
}
extern "C" __global__ void __launch_bounds__(XMR_PREPASS_THREADS)
xmr_mm_split_a(const uint32_t* __restrict__ A, uint8_t* __restrict__ planes, unsigned long long rows, unsigned long long K) {
    split_a_body(A, planes, rows, K);
}
// grouped launches: the R rows from row ro[0] of A
extern "C" __global__ void __launch_bounds__(XMR_PREPASS_THREADS)
xmr_mm_grp_split_a(const unsigned long long* __restrict__ ro, const uint32_t* __restrict__ A, uint8_t* __restrict__ planes,
                   unsigned long long rows, unsigned long long K) {
    split_a_body(A + __ldg(ro) * K, planes, rows, K);
}
// B (u32, batch x K x N, row-major) -> planes[l][b N + n][k] (u8, TRANSPOSED so the MMA's B operand is K-major; a batch's
// products stacked along n).  32 x 32 tiles via smem.
extern "C" __global__ void __launch_bounds__(XMR_PREPASS_THREADS)
xmr_mm_split_bt(const uint32_t* __restrict__ B, uint8_t* __restrict__ planes, unsigned int K, unsigned int N, unsigned int batch) {
    __shared__ uint32_t tile[32][33];
    const unsigned int tiles_n = N / 32u, tiles_k = K / 32u;
    const unsigned long long per = (unsigned long long)tiles_n * tiles_k, n_tiles = per * batch;
    for (unsigned long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const unsigned long long b = t / per;
        const unsigned int w = (unsigned int)(t - b * per), k0 = (w / tiles_n) * 32u, n0 = (w % tiles_n) * 32u;
        const uint32_t* Bb = B + b * K * N;
        for (int i = threadIdx.x; i < 1024; i += 256) tile[i >> 5][i & 31] = __ldg(Bb + (size_t)(k0 + (i >> 5)) * N + n0 + (i & 31));
        __syncthreads();
        const int n = threadIdx.x >> 3, kq = threadIdx.x & 7;      // 32 n x 8 k-quads
        const uint32_t w0 = tile[kq * 4][n], w1 = tile[kq * 4 + 1][n], w2 = tile[kq * 4 + 2][n], w3 = tile[kq * 4 + 3][n];
        const uint32_t lo = __byte_perm(w0, w1, 0x5140u), hi = __byte_perm(w0, w1, 0x7362u);
        const uint32_t lo2 = __byte_perm(w2, w3, 0x5140u), hi2 = __byte_perm(w2, w3, 0x7362u);
        const size_t plane = (size_t)batch * N * K, off = (size_t)(b * N + n0 + n) * K + k0 + kq * 4;
        *reinterpret_cast<uint32_t*>(planes + off) = __byte_perm(lo, lo2, 0x5410u);
        *reinterpret_cast<uint32_t*>(planes + plane + off) = __byte_perm(lo, lo2, 0x7632u);
        *reinterpret_cast<uint32_t*>(planes + 2 * plane + off) = __byte_perm(hi, hi2, 0x5410u);
        *reinterpret_cast<uint32_t*>(planes + 3 * plane + off) = __byte_perm(hi, hi2, 0x7632u);
        __syncthreads();
    }
}

#define XMR_MMTC_KERNEL(NC, INJ)                                                                         \
    extern "C" __global__ void __launch_bounds__(xmr::gemm::CTA_THREADS, 1)                              \
    xmr_mm_u32_tc_nc##NC##_inj##INJ(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap map_a, \
                                    const __grid_constant__ CUtensorMap map_b) {                         \
        xmr::mmtc::body<NC, INJ != 0>(a, &map_a, &map_b);                                                \
    }
XMR_MMTC_KERNEL(1, 0) XMR_MMTC_KERNEL(2, 0) XMR_MMTC_KERNEL(3, 0)
XMR_MMTC_KERNEL(1, 1) XMR_MMTC_KERNEL(2, 1) XMR_MMTC_KERNEL(3, 1)
// grouped (COAST_MM_GROUPED): `ro` = the caller's row offsets, `grp` = the group block the pre-pass wrote (xmr_mm_grp.cuh)
#define XMR_MMTC_GRP_KERNEL(NC, INJ)                                                                     \
    extern "C" __global__ void __launch_bounds__(xmr::gemm::CTA_THREADS, 1)                              \
    xmr_mm_u32_tc_grp_inj##INJ##_nc##NC(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap map_a, \
                                        const __grid_constant__ CUtensorMap map_b, const unsigned long long* ro, const uint8_t* grp) { \
        xmr::mmtc::body<NC, INJ != 0, true>(a, &map_a, &map_b, ro, grp);                                 \
    }
XMR_MMTC_GRP_KERNEL(1, 0) XMR_MMTC_GRP_KERNEL(2, 0) XMR_MMTC_GRP_KERNEL(3, 0)
XMR_MMTC_GRP_KERNEL(1, 1) XMR_MMTC_GRP_KERNEL(2, 1) XMR_MMTC_GRP_KERNEL(3, 1)
// B^T (COAST_MM_B_TRANSPOSED) with a fault plan: only the lazy recompute reads B, so only these differ (the inj0 kernels serve both)
#define XMR_MMTC_BT_KERNEL(NC)                                                                           \
    extern "C" __global__ void __launch_bounds__(xmr::gemm::CTA_THREADS, 1)                              \
    xmr_mm_u32_tc_bt_inj1_nc##NC(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap map_a, \
                                 const __grid_constant__ CUtensorMap map_b) {                            \
        xmr::mmtc::body<NC, true, false, true>(a, &map_a, &map_b);                                       \
    }
XMR_MMTC_BT_KERNEL(1) XMR_MMTC_BT_KERNEL(2) XMR_MMTC_BT_KERNEL(3)
#define XMR_MMTC_BT_GRP_KERNEL(NC)                                                                       \
    extern "C" __global__ void __launch_bounds__(xmr::gemm::CTA_THREADS, 1)                              \
    xmr_mm_u32_tc_bt_grp_inj1_nc##NC(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap map_a, \
                                     const __grid_constant__ CUtensorMap map_b, const unsigned long long* ro, const uint8_t* grp) { \
        xmr::mmtc::body<NC, true, true, true>(a, &map_a, &map_b, ro, grp);                               \
    }
XMR_MMTC_BT_GRP_KERNEL(1) XMR_MMTC_BT_GRP_KERNEL(2) XMR_MMTC_BT_GRP_KERNEL(3)
