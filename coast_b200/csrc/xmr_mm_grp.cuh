// xmr_mm_grp.cuh -- grouped matmuls (COAST_MM_GROUPED): G products that share N and K, product g with its own row count.
//
// The launch holds R = n_units / N stacked rows of A (d_in) and C (d_out) and G dense K x N matrices B (d_aux); `ro` is the
// caller's table of G + 1 u64 row offsets: product g has rows [ro[g], ro[g+1]) of d_in and d_out and the B at d_aux + g K N.
// Every offset is clamped to [ro[0], ro[0] + R] and a decreasing pair counts as zero rows, so a malformed table never reaches
// outside the buffers.  Inside the kernels a row is counted from ro[0] ("local row"); unit = local row * N + column.
//
// The tiled paths cut every product into tiles of TM rows on its own (no tile mixes two products): a one-CTA pre-pass
// (xmr_mm_group_scan) writes tile_start[g], the exclusive scan of ceil(M_g / TM), and the total into the group block in scratch,
// and each tile id finds its product by binary search.  Group block layout (XMR_MM_GRP_*):
//   [0, 128)              TF32 / BF16 only: the A tensor map, rebased by the pre-pass onto row ro[0] of d_in with R rows
//   [128, 128 + 4 (G+1))  tile_start[0 .. G] (u32), tile_start[G] = row tiles of all products
#pragma once
#include "xmr_common.cuh"

namespace xmr {
namespace grp {

// offset of product g, clamped and counted from ro[0]
__device__ __forceinline__ uint32_t clamped_row(const unsigned long long* ro, unsigned long long ro0, uint32_t R, uint32_t g) {
    const unsigned long long o = __ldg(ro + g);
    return o <= ro0 ? 0u : (uint32_t)min(o - ro0, (unsigned long long)R);
}
// rows [start, end) of product g (end >= start)
__device__ __forceinline__ void rows_of(const unsigned long long* ro, unsigned long long ro0, uint32_t R, uint32_t g,
                                        uint32_t& start, uint32_t& end) {
    start = clamped_row(ro, ro0, R, g);
    end = max(start, clamped_row(ro, ro0, R, g + 1u));
}
// the largest g < G with v[g] <= x (v non-decreasing, v[0] <= x)
template <class Load>
__device__ __forceinline__ uint32_t search(uint32_t G, uint32_t x, Load v) {
    uint32_t lo = 0, hi = G;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (v(mid) <= x) lo = mid; else hi = mid;
    }
    return lo;
}

// One tile of a grouped launch: tile id t (of tile_start[G] * tiles_n) -> product g, its rows, and the tile's row-tile tm and
// column-tile tn inside the product in the rasterised order of tile_coords.  An id outside the product (only a malformed table
// gives one) becomes the product's first tile with no rows: it is loaded and computed like any tile, and nothing is stored.
struct Tile { uint32_t g, start, end, tm, tn; };
__device__ __forceinline__ Tile tile_of(const unsigned long long* ro, unsigned long long ro0, uint32_t R, const uint32_t* ts, uint32_t G,
                                        uint32_t tiles_n, uint32_t group_m, uint32_t t) {
    Tile x;
    x.g = search(G, t / tiles_n, [&](uint32_t g) { return __ldg(ts + g); });
    rows_of(ro, ro0, R, x.g, x.start, x.end);
    const uint32_t t0 = __ldg(ts + x.g), tiles_m = __ldg(ts + x.g + 1u) - t0, lt = t - t0 * tiles_n;
    x.tm = x.tn = 0u;
    if (tiles_m == 0u || lt >= tiles_m * tiles_n) {
        x.end = x.start;
    } else {
        const uint32_t per_group = group_m * tiles_n, q = lt / per_group, w = lt - q * per_group;   // xmr::gemm::tile_coords
        const uint32_t rows = min(group_m, tiles_m - q * group_m);
        x.tm = q * group_m + w % rows;
        x.tn = w / rows;
    }
    return x;
}

}  // namespace grp
}  // namespace xmr

// tile_start of a grouped launch (one CTA; G <= XMR_MM_GRP_MAX, so each thread scans at most 1024 entries), and for the GEMM
// kernels the A tensor map: the host encodes its shape, this kernel points it at row ro[0] of `a_base` with R rows
// (tensormap.replace), so a shard or a host-call chunk needs no host-side read of the device table.
extern "C" __global__ void __launch_bounds__(XMR_MM_GRP_SCAN_THREADS)
xmr_mm_group_scan(const unsigned long long* ro, unsigned int G, unsigned int R, unsigned int TM, unsigned int tiles_n,
                  unsigned char* grp, const void* a_base, unsigned int row_bytes, const __grid_constant__ CUtensorMap a_map) {
    __shared__ unsigned int warp_sum[XMR_MM_GRP_SCAN_THREADS / 32];
    unsigned int* ts = reinterpret_cast<unsigned int*>(grp + XMR_MM_GRP_TILES);
    const unsigned long long ro0 = __ldg(ro);
    const unsigned int t = threadIdx.x, lane = t & 31u, w = t >> 5;
    const unsigned int per = (G + XMR_MM_GRP_SCAN_THREADS - 1u) / XMR_MM_GRP_SCAN_THREADS, g0 = min(G, t * per), g1 = min(G, g0 + per);
    // tiles never exceed 2^31 in all (saturating: only a malformed table gets near)
    const unsigned long long cap = 0x7FFFFFFFull / tiles_n;
    unsigned long long mine = 0;
    for (unsigned int g = g0; g < g1; ++g) {
        uint32_t s, e; xmr::grp::rows_of(ro, ro0, R, g, s, e);
        mine += (e - s + TM - 1u) / TM;
    }
    unsigned int v = (unsigned int)min(mine, cap), x = v;
    for (int d = 1; d < 32; d <<= 1) { const unsigned int y = __shfl_up_sync(0xFFFFFFFFu, x, d); if ((int)lane >= d) x = (unsigned int)min((unsigned long long)x + y, cap); }
    if (lane == 31u) warp_sum[w] = x;
    __syncthreads();
    if (w == 0) {
        unsigned int s = warp_sum[lane], y = s;
        for (int d = 1; d < 32; d <<= 1) { const unsigned int z = __shfl_up_sync(0xFFFFFFFFu, y, d); if ((int)lane >= d) y = (unsigned int)min((unsigned long long)y + z, cap); }
        warp_sum[lane] = y - s;                                          // exclusive
    }
    __syncthreads();
    unsigned long long run = (unsigned long long)warp_sum[w] + (x - v);
    for (unsigned int g = g0; g < g1; ++g) {
        ts[g] = (unsigned int)min(run, cap);
        uint32_t s, e; xmr::grp::rows_of(ro, ro0, R, g, s, e);
        run += (e - s + TM - 1u) / TM;
    }
    if (t == XMR_MM_GRP_SCAN_THREADS - 1u) ts[G] = (unsigned int)min(run, cap);
    if (t == 0 && row_bytes) {
        // copy the host's map, rebase it, and release it to the tensor-map proxy of the kernel that follows on the stream
        CUtensorMap* m = reinterpret_cast<CUtensorMap*>(grp);
        const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&a_map);
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(m);
        for (int i = 0; i < 16; ++i) dst[i] = src[i];
        const unsigned long long addr = reinterpret_cast<unsigned long long>(a_base) + ro0 * row_bytes;
        asm volatile("tensormap.replace.tile.global_address.global.b1024.b64 [%0], %1;" ::"l"(m), "l"(addr) : "memory");
        asm volatile("tensormap.replace.tile.global_dim.global.b1024.b32 [%0], 1, %1;" ::"l"(m), "r"(R) : "memory");
        asm volatile("fence.proxy.tensormap::generic.release.gpu;" ::: "memory");
    }
}
