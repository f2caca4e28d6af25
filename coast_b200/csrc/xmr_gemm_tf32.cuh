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
// TF32 wgmma reads both operands K-major, so B goes through a transposing pre-pass (xmr_gemm_bt) into library scratch first.
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, 64 rows of the 128-row tile each.
// Persistent CTAs, one per SM.  Tiles: 128 x 256 unprotected (N % 256 == 0), 128 x 128 otherwise; the accumulators of a
// replica are 64 x 128 wgmma fragments (64 fp32 registers per thread), so TMR holds 192 accumulator registers per thread.
//
// CTA pairs (xmr_gemm_tf32p_*, cluster 2 x 1 x 1): two CTAs compute the two 128-row halves of a 256 x BN tile and share its
// B tile: each CTA loads half of it with a TMA multicast into both CTAs' shared memory, halving the L2 -> SM traffic for B.
// Every element sees the same wgmma sequence as in the single-CTA kernel, so the outputs are bit-identical.
#pragma once
#include "xmr_common.cuh"

namespace xmr {
namespace gemm {

constexpr int BM = 128, BK = 32;                     // BK fp32 = 128 bytes = one swizzle row
constexpr int WG_K = 8;                              // one wgmma consumes 8 tf32 = 32 bytes of K
constexpr int WG_N = 128;                            // wgmma N per instruction
constexpr uint32_t A_STAGE = BM * BK * 4;            // 16 KiB
constexpr int CTA_THREADS = 384;                     // warpgroup 0 = producer, 1-2 = consumers
template <int NC, bool WIDE = (NC == 1)> struct Geom {         // WIDE: 128 x 256 tiles (unprotected, N % 256 == 0)
    static constexpr int BN = WIDE ? 256 : 128;
    static constexpr int NSUB = BN / WG_N;
    static constexpr int STAGES = WIDE ? 4 : 6;                  // 192 KiB of operand stages either way
    static constexpr uint32_t B_STAGE = BK * BN * 4;             // [BN rows of B^T][128 B]
    static constexpr uint32_t SMEM_BYTES = STAGES * (A_STAGE + B_STAGE) + 1024 /*align slack*/ + 256 /*barriers*/;
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

// Epilogue of one consumer thread: vote the NC accumulators of its fragment element by element with the reference's select
// voter / `fcmp oeq`, count, ONE store of the voted value.  Columns [n0 + 128 sub, ...) for sub < nsub_t.
template <int NC, int NSUB, bool INJECT>
__device__ __forceinline__ void epilogue(const xmr_args& a, Tally& tally, float (&acc)[NC][NSUB][64], uint32_t row0, uint32_t n0, uint32_t nsub_t,
                                         bool hints, uint64_t pol_c) {
    const uint32_t flags = a.flags;
    const bool majority = flags & COAST_F_MAJORITY_D;
    float* C = static_cast<float*>(a.out);
    const uint32_t lane = threadIdx.x & 31;
#pragma unroll
    for (int sub = 0; sub < NSUB; ++sub) {
        if ((uint32_t)sub >= nsub_t) break;
#pragma unroll
        for (int j = 0; j < WG_N / 8; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t row = row0 + 8 * h, col = n0 + sub * WG_N + 8 * j + 2 * (lane & 3);
                const unsigned long long local0 = (unsigned long long)row * a.N + col;
                uint32_t o[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int i = 4 * j + 2 * h + e;
                    uint32_t r0 = __float_as_uint(acc[0][sub][i]);
                    uint32_t r1 = NC > 1 ? __float_as_uint(acc[NC > 1 ? 1 : 0][sub][i]) : r0;
                    uint32_t r2 = NC > 2 ? __float_as_uint(acc[NC > 2 ? 2 : 0][sub][i]) : r0;
                    if (INJECT) {
                        Fault f = fault_for_unit(a, NC, local0 + e, [](uint32_t) { return 32u; });
                        if (f.active) {
                            tally.injected++;
                            uint32_t mk = 1u << f.bit;
                            if (f.replica == 0) r0 ^= mk; else if (f.replica == 1) r1 ^= mk; else r2 ^= mk;
                        }
                    }
                    const float f0 = __uint_as_float(r0), f1 = __uint_as_float(r1), f2 = __uint_as_float(r2);
                    uint32_t vote = r0, bad = 0;
                    if (NC == 2) bad = (f0 == f1) ? 0u : 1u;
                    if (NC == 3) {
                        const bool c01 = (f0 == f1), c02 = (f0 == f2);       // fcmp oeq
                        vote = majority ? ((r0 & r1) | (r0 & r2) | (r1 & r2)) : (c01 ? r0 : r2);
                        bad = (c01 && c02) ? 0u : 1u;
                    }
                    o[e] = vote;
                    tally.unit_exit<NC>(bad, 1u, flags, a.unit_base + local0 + e);
                }
                float* dst = C + local0;
                if (hints) st_v2_hint(dst, o[0], o[1], pol_c);
                else *reinterpret_cast<uint2*>(dst) = make_uint2(o[0], o[1]);
            }
        }
    }
}

// PAIR: the CTA pair of a cluster 2 x 1 x 1 computes a 256 x BN tile, rank r the rows [128 r, 128 r + 128); each rank loads half
// of the tile's B^T rows and multicasts them to both, so a stage is released only when the consumers of BOTH CTAs are done with it.
template <int NC, bool INJECT, bool WIDE, bool PAIR>
__device__ __forceinline__ void gemm_body(const xmr_args& a, const CUtensorMap* map_a, const CUtensorMap* map_b) {
    using G = Geom<NC, WIDE>;
    constexpr int BN = G::BN, NSUB = G::NSUB, STAGES = G::STAGES;
    constexpr uint32_t B_STAGE = G::B_STAGE;
    constexpr int B_BOX = PAIR ? 64 : 128;                      // B^T rows per TMA box
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
    const uint32_t tiles_n = a.N / BN, tiles_m = a.M / TM, n_tiles = tiles_m * tiles_n, kblocks = a.K / BK;
    const uint32_t gm1 = (a.mode & 0xFFu) ? (a.mode & 0xFFu) : GROUP_M_DEFAULT;
    const uint32_t group_m = PAIR ? (gm1 > 1u ? gm1 / 2u : 1u) : gm1;   // pair tiles are 256 rows: half as many tile-rows per group
    const bool hints = (a.mode & 0x100u) != 0;
    // Wave quantisation (WIDE only): e.g. 512 tiles on 132 CTAs are 3.9 rounds.  When the last, partial round holds at most half
    // the workers, each of its tiles is split into two 128-column halves, so the tail costs half a round: virtual tile ids
    // [0, sched_full) are whole tiles, [sched_full, n_virtual) are halves (two consecutive ids per tile).
    uint32_t sched_full = n_tiles, n_virtual = n_tiles;
    if (WIDE) {
        const uint32_t whole = (n_tiles / n_workers) * n_workers, rem = n_tiles - whole;
        if (rem && 2u * rem <= n_workers && !(a.mode & 0x200u)) { sched_full = whole; n_virtual = whole + 2u * rem; }
    }
    auto decode = [&](uint32_t v, uint32_t& tm, uint32_t& n_off, uint32_t& bn_t) {
        uint32_t w = v, h = 0, tn;
        bn_t = BN;
        if (v >= sched_full) { w = sched_full + ((v - sched_full) >> 1); h = (v - sched_full) & 1u; bn_t = BN / 2; }
        tile_coords(w, tiles_m, tiles_n, group_m, tm, tn);
        n_off = tn * BN + h * (BN / 2);
    };

    if (threadIdx.x == 0) {
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
                decode(tile, tm, n_off, bn_t);
                const int m0 = (int)(tm * TM + rank * BM);
                const uint32_t rows_b = bn_t / CTAS;                // B^T rows this CTA loads (for both CTAs of a pair)
                for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
                    const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                    mbar_wait_or_trap(&empty[s], ph ^ 1u);
                    mbar_arrive_expect_tx(&full[s], A_STAGE + bn_t * BK * 4u);
                    tma_load_2d_hint(sA + s * A_STAGE, map_a, &full[s], (int)(kb * BK), m0, pol_a);          // box {32 k, 128 m}
                    for (uint32_t c = 0; c < rows_b / B_BOX; ++c) {
                        const uint32_t r = rank * rows_b + c * B_BOX;                                        // row of the tile's B^T
                        if (PAIR) tma_load_2d_mcast(sB + s * B_STAGE + r * 128u, map_b, &full[s], (int)(kb * BK), (int)(n_off + r), (uint16_t)3, pol_b);
                        else tma_load_2d_hint(sB + s * B_STAGE + r * 128u, map_b, &full[s], (int)(kb * BK), (int)(n_off + r), pol_b);
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
        float acc[NC][NSUB][64];
        uint32_t it = 0;
        for (uint32_t tile = worker; tile < n_virtual; tile += n_workers) {
            uint32_t tm, n0, bn_t;
            decode(tile, tm, n0, bn_t);
            const uint32_t nsub_t = bn_t / WG_N;
#pragma unroll
            for (int r = 0; r < NC; ++r)
#pragma unroll
                for (int sub = 0; sub < NSUB; ++sub)
#pragma unroll
                    for (int i = 0; i < 64; ++i) acc[r][sub][i] = 0.f;
#pragma unroll
            for (int r = 0; r < NC; ++r)
#pragma unroll
                for (int sub = 0; sub < NSUB; ++sub) wg_fence_regs(acc[r][sub]);
            for (uint32_t kb = 0; kb < kblocks; ++kb, ++it) {
                const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                mbar_wait_or_trap(&full[s], ph);
                const uint64_t da0 = wg_desc(smem_u32(sA + s * A_STAGE) + a_off), db0 = wg_desc(smem_u32(sB + s * B_STAGE));
                wg_fence();
#pragma unroll
                for (int k = 0; k < BK / WG_K; ++k) {
#pragma unroll
                    for (int sub = 0; sub < NSUB; ++sub) {
                        if ((uint32_t)sub >= nsub_t) break;
                        const uint64_t da = da0 + (uint64_t)(2 * k), db = db0 + (uint64_t)(2 * k + sub * (WG_N * 128 >> 4));
#pragma unroll
                        for (int r = 0; r < NC; ++r) {
                            // with several replica accumulators in flight, ptxas may move one between the asynchronous wgmmas
                            // (seen on the DWC kernel: wrong results); retiring each replica's wgmma before the next keeps them apart
                            if (NC > 1 && r > 0) { wg_commit(); wg_wait<0>(); wg_fence(); }
                            wgmma_tf32_m64n128k8(acc[r][sub], da, db);
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
            const uint32_t row0 = tm * TM + rank * BM + (uint32_t)(wg - 1) * 64u + 16u * (t >> 5) + ((t & 31) >> 2);
            epilogue<NC, NSUB, INJECT>(a, tally, acc, row0, n0, nsub_t, hints, pol_c);
        }
        tally.flush(a.counters);
    }
    if (PAIR) cluster_sync_all();                               // nobody leaves while the peer's multicasts / remote arrivals are in flight
}

}  // namespace gemm
}  // namespace xmr

// B (K x N, row-major) -> B^T (N x K): the K-major operand TF32 wgmma reads.  32 x 32 tiles through shared memory.
extern "C" __global__ void __launch_bounds__(256)
xmr_gemm_bt(const float* __restrict__ B, float* __restrict__ Bt, unsigned int K, unsigned int N) {
    __shared__ float tile[32][33];
    const unsigned int tiles_n = N / 32u, tiles_k = K / 32u;
    for (unsigned int t = blockIdx.x; t < tiles_n * tiles_k; t += gridDim.x) {
        const unsigned int k0 = (t / tiles_n) * 32u, n0 = (t % tiles_n) * 32u;
        for (int i = threadIdx.x; i < 1024; i += 256) tile[i >> 5][i & 31] = __ldg(B + (size_t)(k0 + (i >> 5)) * N + n0 + (i & 31));
        __syncthreads();
        for (int i = threadIdx.x; i < 1024; i += 256) Bt[(size_t)(n0 + (i >> 5)) * K + k0 + (i & 31)] = tile[i & 31][i >> 5];
        __syncthreads();
    }
}

#define XMR_GEMM_KERNEL(NAME, NC, INJ, WIDE, PAIR, CLUSTER)                                              \
    extern "C" __global__ void CLUSTER __launch_bounds__(xmr::gemm::CTA_THREADS, 1)                      \
    NAME(const __grid_constant__ xmr_args a, const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b) { \
        xmr::gemm::gemm_body<NC, INJ != 0, WIDE, PAIR>(a, &map_a, &map_b);                               \
    }
#define XMR_NO_CLUSTER
#define XMR_PAIR_CLUSTER __cluster_dims__(2, 1, 1)
XMR_GEMM_KERNEL(xmr_gemm_tf32_nc1_inj0, 1, 0, true, false, XMR_NO_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32_nc2_inj0, 2, 0, false, false, XMR_NO_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32_nc3_inj0, 3, 0, false, false, XMR_NO_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32_nc1_inj1, 1, 1, true, false, XMR_NO_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32_nc2_inj1, 2, 1, false, false, XMR_NO_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32_nc3_inj1, 3, 1, false, false, XMR_NO_CLUSTER)
// unprotected, N a multiple of 128 but not of 256: 128 x 128 tiles
XMR_GEMM_KERNEL(xmr_gemm_tf32n_nc1_inj0, 1, 0, false, false, XMR_NO_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32n_nc1_inj1, 1, 1, false, false, XMR_NO_CLUSTER)
// CTA pairs: 256 x 256 (unprotected) / 256 x 128 pair tiles
XMR_GEMM_KERNEL(xmr_gemm_tf32p_nc1_inj0, 1, 0, true, true, XMR_PAIR_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32p_nc2_inj0, 2, 0, false, true, XMR_PAIR_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32p_nc3_inj0, 3, 0, false, true, XMR_PAIR_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32p_nc1_inj1, 1, 1, true, true, XMR_PAIR_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32p_nc2_inj1, 2, 1, false, true, XMR_PAIR_CLUSTER)
XMR_GEMM_KERNEL(xmr_gemm_tf32p_nc3_inj1, 3, 1, false, true, XMR_PAIR_CLUSTER)
