// xmr_mm.cuh -- protected integer matrix multiply (tests/mm_common/mm_common_tmr.c:3-20 and
// tests/matrixMultiply/matrixMultiply.c:95-112 of byuccl/coast), exact modulo 2^32.
//
// Unit = one element r[i][j] = sum_k f[i][k]*s[k][j].  The reference accumulates in an
// `unsigned long` and truncates on the store (:16 / :108); only the low 32 bits are observable,
// so each replica keeps `sum` mod 2^32.  SoR exit = that element store: ONE mm_t vote per unit.
// Fault sites: s in [0,K): `sum` after k-step s (32 bits).
//
// Layout: NC replica lanes per element, (32/NC) consecutive j per warp -> B rows are read
// coalesced, the A element is a warp-broadcast; replicas of an element share every load
// (same address -> one L1 transaction).
//
// Grouped launches (COAST_MM_GROUPED, xmr_mm_grp.cuh): each element finds its row's product by binary search over the row
// offsets; a row outside every product's clamped range (a malformed table) is neither computed nor stored.
// BT (COAST_MM_B_TRANSPOSED): aux holds B^T, N rows of K per product; element (k, j) is read at j*K + k instead of k*N + j.
#pragma once
#include "xmr_common.cuh"
#include "xmr_mm_grp.cuh"

namespace xmr {

template <int NC, bool INJECT, bool GROUPED = false, bool BT = false>
__device__ __forceinline__ void mm_u32_body(const xmr_args& a, const unsigned long long* ro = nullptr) {
    constexpr int UPW = Lanes<NC>::kUnitsPerWarp;
    const int lane = threadIdx.x & 31;
    const int r = Lanes<NC>::replica(lane);
    const unsigned long long gwarp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long nwarps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long n_wtiles = (a.n_units + UPW - 1) / UPW;
    const uint32_t* __restrict__ A = static_cast<const uint32_t*>(a.in);
    const uint32_t* __restrict__ B = static_cast<const uint32_t*>(a.aux);
    uint32_t* C = static_cast<uint32_t*>(a.out);
    const uint32_t K = a.K, N = a.N;
    const unsigned long long ro0 = GROUPED ? __ldg(ro) : 0ull;
    const uint32_t R = GROUPED ? (uint32_t)(a.n_units / N) : 0u;
    if constexpr (GROUPED) C += ro0 * N;                        // rows counted from ro[0]
    Tally tally(a);
    for (unsigned long long wt = gwarp; wt < n_wtiles; wt += nwarps) {
        const unsigned long long local = wt * UPW + Lanes<NC>::unit(lane);
        bool valid = local < a.n_units;
        const unsigned long long e = valid ? local : 0ull;
        const uint32_t i = (uint32_t)(e / N), j = (uint32_t)(e % N);
        uint32_t g = 0;
        if constexpr (GROUPED) {                                 // the product of row i: the last one starting at or before it
            g = grp::search(a.M, i, [&](uint32_t x) { return grp::clamped_row(ro, ro0, R, x); });
            uint32_t s, end; grp::rows_of(ro, ro0, R, g, s, end);
            valid = valid && i >= s && i < end;
        }
        uint32_t fsite = 0xFFFFFFFFu, fmask = 0u;
        if (INJECT) {
            Fault f = fault_for_unit(a, NC, e, [](uint32_t) { return 32u; });
            if (f.active && valid) {
                if (Lanes<NC>::voter(lane)) tally.injected++;
                if ((int)f.replica == r) { fsite = f.site; fmask = 1u << f.bit; }
            }
        }
        const uint32_t* ap = A + (size_t)(ro0 + i) * K;         // i: row of the stacked problem; a batch's product i / M
        const uint32_t* bp = B + (size_t)(GROUPED ? g : i / a.M) * K * N + (BT ? (size_t)j * K : j);
        const size_t bstride = BT ? 1u : N;                     // from B[k][j] to B[k + 1][j]
        uint32_t sum = 0;
        if (!(a.flags & XMR_F_STORE_VOTES)) {
            for (uint32_t k = 0; k < K; ++k) {                  // :12-14
                sum += __ldg(ap + k) * __ldg(bp + k * bstride);
                if (INJECT && fsite == k) sum ^= fmask;
            }
            Voted v = vote_u32<NC, 4>(sum, a.flags & COAST_F_MAJORITY_VOTER);
            if (valid && Lanes<NC>::voter(lane)) {
                C[local] = v.vote;                              // :16
                tally.unit_exit<NC>(v.bad, 1u, a.flags, a.unit_base + local);
            }
        } else {
            // -storeDataSync / -noMemReplication: `sum += ...` (:13) is voted at every k, the replicas continue with the voted
            // value; K votes + the SoR-exit store (:16)
            const bool majority = a.flags & COAST_F_MAJORITY_VOTER;
            uint32_t bad = 0;
            for (uint32_t k = 0; k < K; ++k) {
                sum += __ldg(ap + k) * __ldg(bp + k * bstride);
                bad += store_vote<NC>(sum, lane, majority);
                if (INJECT && fsite == k) sum ^= fmask;
            }
            bad += store_vote<NC>(sum, lane, majority);
            if (valid && Lanes<NC>::voter(lane)) {
                C[local] = sum;
                tally.unit_exit<NC>(bad, K + 1u, a.flags, a.unit_base + local);
            }
        }
    }
    tally.flush(a.counters);
}

}  // namespace xmr

#define XMR_MM_KERNEL(NC, INJ)                                                                           \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_mm_u32_nc##NC##_inj##INJ(const __grid_constant__ xmr_args a) { xmr::mm_u32_body<NC, INJ != 0>(a); }
XMR_MM_KERNEL(1, 0) XMR_MM_KERNEL(2, 0) XMR_MM_KERNEL(3, 0)
XMR_MM_KERNEL(1, 1) XMR_MM_KERNEL(2, 1) XMR_MM_KERNEL(3, 1)
// grouped (COAST_MM_GROUPED): `ro` = the caller's row offsets (no pre-pass)
#define XMR_MM_GRP_KERNEL(NC, INJ)                                                                       \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_mm_u32_grp_inj##INJ##_nc##NC(const __grid_constant__ xmr_args a, const unsigned long long* ro) { \
        xmr::mm_u32_body<NC, INJ != 0, true>(a, ro);                                                     \
    }
XMR_MM_GRP_KERNEL(1, 0) XMR_MM_GRP_KERNEL(2, 0) XMR_MM_GRP_KERNEL(3, 0)
XMR_MM_GRP_KERNEL(1, 1) XMR_MM_GRP_KERNEL(2, 1) XMR_MM_GRP_KERNEL(3, 1)
// B^T (COAST_MM_B_TRANSPOSED), uniform / batched and grouped
#define XMR_MM_BT_KERNEL(NC, INJ)                                                                        \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_mm_u32_bt_inj##INJ##_nc##NC(const __grid_constant__ xmr_args a) { xmr::mm_u32_body<NC, INJ != 0, false, true>(a); }
XMR_MM_BT_KERNEL(1, 0) XMR_MM_BT_KERNEL(2, 0) XMR_MM_BT_KERNEL(3, 0)
XMR_MM_BT_KERNEL(1, 1) XMR_MM_BT_KERNEL(2, 1) XMR_MM_BT_KERNEL(3, 1)
#define XMR_MM_BT_GRP_KERNEL(NC, INJ)                                                                    \
    extern "C" __global__ void __launch_bounds__(XMR_CTA_THREADS)                                        \
    xmr_mm_u32_bt_grp_inj##INJ##_nc##NC(const __grid_constant__ xmr_args a, const unsigned long long* ro) { \
        xmr::mm_u32_body<NC, INJ != 0, true, true>(a, ro);                                               \
    }
XMR_MM_BT_GRP_KERNEL(1, 0) XMR_MM_BT_GRP_KERNEL(2, 0) XMR_MM_BT_GRP_KERNEL(3, 0)
XMR_MM_BT_GRP_KERNEL(1, 1) XMR_MM_BT_GRP_KERNEL(2, 1) XMR_MM_BT_GRP_KERNEL(3, 1)
