// xmr_common.cuh -- device-side building blocks of the redundant-execution engine (sm_90a).
//
//   replica layout : NC (1/2/3) replicas of a unit sit on ADJACENT LANES of one warp
//                    (lane = NC*u + r).  This is the analogue of cloneInsns putting I.DWC/I.TMR
//                    right after I (projects/dataflowProtection/cloning.cpp:2189-2204) with
//                    register-resident replica state = replicated memory (rule D1, passes.rst:329).
//   voter          : reference SELECT voter, vote = (r0 == r1) ? r0 : r2
//                    (synchronization.cpp:512-522; same shape at :439-448, :631-642, :934-938),
//                    built from __shfl_down_sync; per-element-type granularity (u8/u16/u32/f32).
//   error counter  : +1 per voted element with !(r0==r1 && r0==r2) (synchronization.cpp:1391-1431),
//                    accumulated per lane, __reduce_add_sync per warp, one atomicAdd per warp.
//   DWC            : r0 != r1 on any element of the unit -> dwc_detected++ (synchronization.cpp:1117-1192).
//   injector       : Philox4x32-10 keyed single-bit flip (simulation/platform/resources/injector.py:202-207).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/coast_rt.h"   // COAST_F_*, COAST_AES_*
#include "xmr_args.h"
#include "xmr_geom.h"

namespace xmr {

// ---------------------------------------------------------------- Philox4x32-10
struct u4 { uint32_t x, y, z, w; };

__device__ __forceinline__ u4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return u4{c0, c1, c2, c3};
}

// ---------------------------------------------------------------- fault decision
struct Fault { bool active; uint32_t replica, site, bit; };

// `width(site)` is the bit width of the value living at `site` (kernel-specific functor).
template <class WidthFn>
__device__ __forceinline__ Fault fault_for_unit(const xmr_args& a, uint32_t nc, uint64_t local, WidthFn width) {
    Fault f{false, 0, 0, 0};
    if (a.plan_mode == 1u) {
        uint64_t g = a.unit_base + local;
        u4 x = philox4x32_10((uint32_t)g, (uint32_t)(g >> 32), 0u, 0u, a.seed_lo, a.seed_hi);
        if (x.x < a.threshold) {
            f.replica = x.y % nc;
            f.site = x.z % a.n_sites;
            f.bit = x.w % width(f.site);
            f.active = true;
        }
    } else if (a.plan_mode == 2u) {
        uint32_t e = __ldg(a.plan_table + local);
        uint32_t rep = (e >> 29) & 3u, site = (e >> 5) & 0xFFFFFFu, bit = e & 31u;
        if ((e & 0x80000000u) && rep < nc && site < a.n_sites && bit < width(site)) {
            f.replica = rep; f.site = site; f.bit = bit; f.active = true;
        }
    }
    return f;
}

// The same decision with a per-unit site count (ragged batches: each unit has its own length).  A unit without sites is never
// injected, and the Bernoulli draw is not taken modulo zero.
template <class WidthFn>
__device__ __forceinline__ Fault fault_for_unit(const xmr_args& a, uint32_t nc, uint64_t local, uint32_t n_sites, WidthFn width) {
    Fault f{false, 0, 0, 0};
    if (n_sites == 0u) return f;
    if (a.plan_mode == 1u) {
        uint64_t g = a.unit_base + local;
        u4 x = philox4x32_10((uint32_t)g, (uint32_t)(g >> 32), 0u, 0u, a.seed_lo, a.seed_hi);
        if (x.x < a.threshold) {
            f.replica = x.y % nc;
            f.site = x.z % n_sites;
            f.bit = x.w % width(f.site);
            f.active = true;
        }
    } else if (a.plan_mode == 2u) {
        uint32_t e = __ldg(a.plan_table + local);
        uint32_t rep = (e >> 29) & 3u, site = (e >> 5) & 0xFFFFFFu, bit = e & 31u;
        if ((e & 0x80000000u) && rep < nc && site < n_sites && bit < width(site)) {
            f.replica = rep; f.site = site; f.bit = bit; f.active = true;
        }
    }
    return f;
}

// ---------------------------------------------------------------- lane geometry
template <int NC> struct Lanes {
    static constexpr int kUnitsPerWarp = 32 / NC;           // 32, 16, 10 (lanes 30,31 idle under TMR)
    // replica index and unit-in-warp of this lane; the 2 spare TMR lanes shadow unit 9 and never vote
    __device__ static __forceinline__ int replica(int lane) { return NC == 3 ? (lane >= 30 ? lane - 30 : lane % 3) : lane % NC; }
    __device__ static __forceinline__ int unit(int lane) { return NC == 3 ? (lane >= 30 ? 9 : lane / 3) : lane / NC; }
    __device__ static __forceinline__ bool voter(int lane) { return NC == 3 ? (lane < 30 && lane % 3 == 0) : (lane % NC == 0); }
};

// ---------------------------------------------------------------- voters
// Result of voting one 32-bit register that packs `EB`-byte elements (EB = 1, 2 or 4).
//   vote : the value the SoR-exit store writes
//   bad  : number of packed elements with !(r0==r1 && r0==r2)   (TMR)  /  r0!=r1 (DWC)
struct Voted { uint32_t vote; uint32_t bad; };

template <int EB> __device__ __forceinline__ uint32_t eq_mask(uint32_t a, uint32_t b) {
    if (EB == 1) return __vcmpeq4(a, b);           // 0xFF per equal byte
    if (EB == 2) return __vcmpeq2(a, b);           // 0xFFFF per equal half
    return a == b ? 0xFFFFFFFFu : 0u;
}

// Must be called by ALL lanes of the warp (shuffles); only lanes with Lanes<NC>::voter() hold a
// meaningful result.  `x` is this lane's replica value.
template <int NC, int EB>
__device__ __forceinline__ Voted vote_u32(uint32_t x, bool majority) {
    Voted v{x, 0u};
    if (NC == 1) return v;
    uint32_t r1 = __shfl_down_sync(0xFFFFFFFFu, x, 1);
    if (NC == 2) {
        uint32_t ne = ~eq_mask<EB>(x, r1);
        v.bad = __popc(ne) / (8 * EB);
        return v;                                   // the original's store proceeds with r0
    }
    uint32_t r2 = __shfl_down_sync(0xFFFFFFFFu, x, 2);
    uint32_t e01 = eq_mask<EB>(x, r1), e02 = eq_mask<EB>(x, r2);
    v.vote = majority ? ((x & r1) | (x & r2) | (r1 & r2)) : ((x & e01) | (r2 & ~e01));
    v.bad = __popc(~(e01 & e02)) / (8 * EB);
    return v;
}

// fp32 voter with the reference's `fcmp oeq` (synchronization.cpp:57-62): NaN != NaN, +0 == -0.
template <int NC>
__device__ __forceinline__ Voted vote_f32(float x, bool majority) {
    uint32_t xb = __float_as_uint(x);
    Voted v{xb, 0u};
    if (NC == 1) return v;
    float r1 = __shfl_down_sync(0xFFFFFFFFu, x, 1);
    if (NC == 2) { v.bad = (x == r1) ? 0u : 1u; return v; }
    float r2 = __shfl_down_sync(0xFFFFFFFFu, x, 2);
    bool c01 = (x == r1), c02 = (x == r2);
    uint32_t b1 = __float_as_uint(r1), b2 = __float_as_uint(r2);
    v.vote = majority ? ((xb & b1) | (xb & b2) | (b1 & b2)) : (c01 ? xb : b2);
    v.bad = (c01 && c02) ? 0u : 1u;
    return v;
}

// In-loop store vote (-storeDataSync / -noMemReplication, synchronization.cpp:476-560): every lane of the unit reads all
// NC copies, so -- unlike vote_u32 -- ALL replica lanes hold the result and, under TMR, continue with the voted value
// (:519-529 hands `sel` to the three stores).  DWC keeps its own value (the reference would have aborted).  Returns 1 if
// the copies disagree.  Must be called by all 32 lanes; `x` is a value of at most 32 bits.
template <int NC>
__device__ __forceinline__ uint32_t store_vote(uint32_t& x, int lane, bool majority) {
    if (NC == 1) return 0u;
    const int base = Lanes<NC>::unit(lane) * NC;
    const uint32_t r0 = __shfl_sync(0xFFFFFFFFu, x, base), r1 = __shfl_sync(0xFFFFFFFFu, x, base + 1);
    if (NC == 2) return r0 != r1 ? 1u : 0u;
    const uint32_t r2 = __shfl_sync(0xFFFFFFFFu, x, base + 2);
    const bool c01 = r0 == r1, c02 = r0 == r2;
    x = majority ? ((r0 & r1) | (r0 & r2) | (r1 & r2)) : (c01 ? r0 : r2);
    return (c01 && c02) ? 0u : 1u;
}

// Same for a register that packs up to four u8 elements in its TOP `nb` bytes (a big-endian-packed message word): one vote per
// byte, returns the number of disagreeing bytes among those nb.
template <int NC>
__device__ __forceinline__ uint32_t store_vote_bytes(uint32_t& x, uint32_t nb, int lane, bool majority) {
    if (NC == 1 || nb == 0u) return 0u;
    const uint32_t live = 0xFFFFFFFFu << (8u * (4u - nb));
    const int base = Lanes<NC>::unit(lane) * NC;
    const uint32_t r0 = __shfl_sync(0xFFFFFFFFu, x, base), r1 = __shfl_sync(0xFFFFFFFFu, x, base + 1);
    const uint32_t e01 = __vcmpeq4(r0, r1);
    if (NC == 2) return __popc(~e01 & live) >> 3;
    const uint32_t r2 = __shfl_sync(0xFFFFFFFFu, x, base + 2);
    const uint32_t e02 = __vcmpeq4(r0, r2);
    x = majority ? ((r0 & r1) | (r0 & r2) | (r1 & r2)) : ((r0 & e01) | (r2 & ~e01));
    return __popc(~(e01 & e02) & live) >> 3;
}

// ---------------------------------------------------------------- per-thread tallies -> counters
struct Tally {
    uint32_t errors = 0, dwc = 0, syncs = 0, injected = 0;
    unsigned long long first = ~0ull;
    unsigned char* status = nullptr;          // optional per-unit disagreement count (campaign tooling)
    unsigned long long base = 0;
    __device__ __forceinline__ Tally() {}
    __device__ __forceinline__ explicit Tally(const xmr_args& a) : status(a.status), base(a.unit_base) {}
    // one unit's SoR exit: `bad` disagreeing elements out of `nvotes`
    template <int NC> __device__ __forceinline__ void unit_exit(uint32_t bad, uint32_t nvotes, uint32_t flags, unsigned long long gunit) {
        if (NC == 3) {
            if (flags & COAST_F_COUNT_ERRORS) {
                errors += bad;
                if (flags & COAST_F_COUNT_SYNCS) syncs += nvotes;     // synchronization.cpp:1415-1425
            }
        } else if (NC == 2) {
            dwc += bad ? 1u : 0u;
        }
        if (NC > 1 && bad && gunit < first) first = gunit;
        if (status) status[gunit - base] = (unsigned char)(NC > 1 ? (bad > 255u ? 255u : bad) : 0u);
    }
    // all 32 lanes must call
    __device__ __forceinline__ void flush(unsigned long long* ctr) {
        uint32_t e = __reduce_add_sync(0xFFFFFFFFu, errors);
        uint32_t d = __reduce_add_sync(0xFFFFFFFFu, dwc);
        uint32_t s = __reduce_add_sync(0xFFFFFFFFu, syncs);
        uint32_t j = __reduce_add_sync(0xFFFFFFFFu, injected);
        uint32_t fhi = __reduce_min_sync(0xFFFFFFFFu, (uint32_t)(first >> 32));
        uint32_t flo = __reduce_min_sync(0xFFFFFFFFu, (uint32_t)(first >> 32) == fhi ? (uint32_t)first : 0xFFFFFFFFu);
        if ((threadIdx.x & 31) == 0) {
            // system scope: the block may be ANOTHER GPU's, mapped over NVLink (coast_counters_attach) -- the multi-GPU fold
            if (e) atomicAdd_system(ctr + XMR_CTR_ERRORS, (unsigned long long)e);
            if (d) atomicAdd_system(ctr + XMR_CTR_DWC, (unsigned long long)d);
            if (s) atomicAdd_system(ctr + XMR_CTR_SYNCS, (unsigned long long)s);
            if (j) atomicAdd_system(ctr + XMR_CTR_INJECTED, (unsigned long long)j);
            unsigned long long f = ((unsigned long long)fhi << 32) | flo;
            if (f != ~0ull) atomicMin_system(ctr + XMR_CTR_FIRST, f);
        }
    }
};

// ---------------------------------------------------------------- mbarrier / TMA (sm_90 PTX; SASS UTMALDG / SYNCS)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 2-D tiled TMA load: box {inner, rows} at coordinates (c0 = inner element, c1 = row)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// ---------------------------------------------------------------- TMA tile ring
// A CTA-wide 2-stage ring of input tiles: TILE_ROWS rows of ROW_BYTES bytes, filled by thread 0 with
// LOADS equal tiled TMA loads of <= 256 rows (box = {ROW_BYTES, TILE_ROWS/LOADS}; rows past the end of
// the tensor are zero-filled by the hardware, which is what makes ragged tails free).
//   prologue : ring.init(smem, tmap); ring.issue(0, first_tile)
//   loop it  : ring.issue((it+1)&1, next_tile)  [if any];  ring.wait(it);  <copy rows to registers>;
//              __syncthreads();   // everyone drained stage it&1 -> it may be refilled at it+1
template <int TILE_ROWS, int ROW_BYTES>
struct TileRing {
    static constexpr int LOADS = (int)xmr_ring_loads(TILE_ROWS);
    static constexpr int BOX_ROWS = TILE_ROWS / LOADS;
    static_assert(TILE_ROWS % LOADS == 0 && BOX_ROWS <= 256, "tile must split into equal TMA boxes");
    static constexpr uint32_t TILE_BYTES = (uint32_t)TILE_ROWS * ROW_BYTES;
    static constexpr uint32_t STAGE_STRIDE = xmr_ring_stride(TILE_ROWS, ROW_BYTES);
    static constexpr uint32_t SMEM_BYTES = xmr_ring_smem(XMR_STAGES, TILE_ROWS, ROW_BYTES, XMR_RING_TAIL);
    static_assert(XMR_STAGES * sizeof(uint64_t) <= XMR_RING_TAIL, "the full barriers fit behind the tiles");
    uint8_t* tiles;
    uint64_t* full;
    const CUtensorMap* tmap;
    // The host may describe the same dense bytes with rows 2^pack_shift times longer (box {ROW_BYTES << s, BOX_ROWS >> s}):
    // identical shared-memory image, fewer and larger requests -- what matters when the tensor lives in mapped HOST memory
    // and every row is its own PCIe read (16-byte AES rows: r02 zero-copy experiment).
    uint32_t pack_shift = 0;
    __device__ __forceinline__ void init(uint8_t* smem, const CUtensorMap* map, uint32_t row_pack_shift = 0) {
        pack_shift = row_pack_shift;
        tiles = smem;
        full = reinterpret_cast<uint64_t*>(smem + XMR_STAGES * STAGE_STRIDE);
        tmap = map;
        if (threadIdx.x == 0) {
            tma_prefetch_desc(map);
#pragma unroll
            for (int s = 0; s < XMR_STAGES; ++s) mbar_init(&full[s], 1);
            fence_barrier_init();
        }
        __syncthreads();
    }
    __device__ __forceinline__ void issue(uint32_t stage, uint32_t tile) {
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(&full[stage], TILE_BYTES);
#pragma unroll
            for (int l = 0; l < LOADS; ++l)
                tma_load_2d(tiles + stage * STAGE_STRIDE + l * BOX_ROWS * ROW_BYTES, tmap, &full[stage], 0,
                            (int)((tile * TILE_ROWS + l * BOX_ROWS) >> pack_shift));
        }
    }
    __device__ __forceinline__ const uint8_t* wait(uint32_t it) {
        mbar_wait(&full[it & 1u], (it >> 1) & 1u);
        return tiles + (it & 1u) * STAGE_STRIDE;
    }
};

}  // namespace xmr
