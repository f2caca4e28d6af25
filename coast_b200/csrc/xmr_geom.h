/*
 * xmr_geom.h -- launch geometry shared by the host runtime (coast_rt.c, plain C) and the kernels (coast_kernels.cu).
 *
 * Every CTA size, tile height and dynamic shared-memory size the host launches with is stated here once.  The kernels
 * define their layouts from the same functions and static_assert that each layout fits the size the host passes, so a
 * tuning change (stages, tile width, ring depth, CTA size) is made in one place and a mismatch stops the build.
 * All sizes are in bytes; `nc` is the replica count (1, 2 or 3).
 */
#ifndef XMR_GEOM_H_
#define XMR_GEOM_H_

#ifdef __CUDACC__
#define XMR_GEOM_FN static constexpr __host__ __device__ inline
#else
#define XMR_GEOM_FN static inline
#endif

/* ---- TMA tile ring: `stages` tiles of tile_rows x row_bytes, each 1 KiB aligned, then `tail` bytes of mbarriers ---- */
XMR_GEOM_FN unsigned xmr_align(unsigned x, unsigned a) { return (x + a - 1u) & ~(a - 1u); }
XMR_GEOM_FN unsigned xmr_ring_stride(unsigned tile_rows, unsigned row_bytes) { return xmr_align(tile_rows * row_bytes, 1024u); }
XMR_GEOM_FN unsigned xmr_ring_smem(unsigned stages, unsigned tile_rows, unsigned row_bytes, unsigned tail) {
    return stages * xmr_ring_stride(tile_rows, row_bytes) + tail;
}
/* smallest number of equal TMA boxes of at most 256 rows a tile splits into */
XMR_GEOM_FN unsigned xmr_ring_loads(unsigned tile_rows) {
    unsigned l = (tile_rows + 255u) / 256u;
    while (tile_rows % l) ++l;
    return l;
}
XMR_GEOM_FN unsigned xmr_units_per_warp(unsigned nc) { return 32u / nc; }

/* ---- lane-interleaved kernels (SHA-256, CRC16 and matmul general paths, CHStone sha) and the SHA-256 64-byte ring ---- */
#define XMR_CTA_THREADS 256
#define XMR_WARPS       8
#define XMR_STAGES      2
#define XMR_RING_TAIL   64u                  /* TileRing: XMR_STAGES full barriers */
XMR_GEOM_FN unsigned xmr_sha_tile_rows(unsigned nc) { return XMR_WARPS * xmr_units_per_warp(nc); }
XMR_GEOM_FN unsigned xmr_sha_smem(unsigned nc) { return xmr_ring_smem(XMR_STAGES, xmr_sha_tile_rows(nc), 64u, XMR_RING_TAIL); }

/* SHA-256 TMR, segmented layout: 4 groups of 3 replica warps, one 32-message row block per group; after the ring, an
 * exchange buffer [tile parity 2][group 4][replica 1..2][8 state words][32 lanes] of u32 */
#define XMR_SHA_SEG_THREADS    384
#define XMR_SHA_SEG_TILE_ROWS  128u
#define XMR_SHA_SEG_EXCH_BYTES (2u * 4u * 2u * 8u * 32u * 4u)
XMR_GEOM_FN unsigned xmr_sha_seg_exch_offset(void) {
    return xmr_align(xmr_ring_smem(XMR_STAGES, XMR_SHA_SEG_TILE_ROWS, 64u, XMR_RING_TAIL), 128u);
}
XMR_GEOM_FN unsigned xmr_sha_seg_smem(void) { return xmr_sha_seg_exch_offset() + XMR_SHA_SEG_EXCH_BYTES; }

/* ---- CRC16 table kernel: shared window = [.., 0x10000) unused | 64 KiB byte-step table | tile ring at 0x20000 ---- */
#define XMR_CRC_TAB  0x10000u
#define XMR_CRC_RING 0x20000u
XMR_GEOM_FN unsigned xmr_crc_threads(unsigned nc) { return nc == 1u ? 768u : 1024u; }   /* 768: the 64 B x 1024 tile would not fit */
XMR_GEOM_FN unsigned xmr_crc_tile_rows(unsigned nc) { return xmr_crc_threads(nc) / 32u * xmr_units_per_warp(nc); }
XMR_GEOM_FN unsigned xmr_crc_smem(unsigned nc) { return XMR_CRC_RING + xmr_ring_smem(XMR_STAGES, xmr_crc_tile_rows(nc), 64u, XMR_RING_TAIL); }

/* ---- AES-128 and CHStone aes: 512-thread CTAs; shared window = ring + queues | T01 at 0x10000 | T23 at 0x20000 |
 * decrypt only: (InvS, S) at 0x30000, 32 KiB ---- */
#define XMR_AES_THREADS 512
#define XMR_AES_WARPS   16
#define XMR_AES_TAB01   0x10000u
#define XMR_AES_TAB23   0x20000u
#define XMR_AES_SIS     0x30000u
XMR_GEOM_FN unsigned xmr_aes_blocks_per_lane(unsigned nc) { return nc == 1u ? 2u : 4u; }
XMR_GEOM_FN unsigned xmr_aes_tile_rows(unsigned nc) { return XMR_AES_WARPS * xmr_units_per_warp(nc) * xmr_aes_blocks_per_lane(nc); }
XMR_GEOM_FN unsigned xmr_aes_smem(int dec) { return dec ? XMR_AES_SIS + 0x8000u : XMR_AES_SIS; }

/* ---- exact integer matmul, register-tiled: BM x BN x BK tiles, nc x VT threads (replicas on adjacent warps) ---- */
#define XMR_MMT_BM 64u
#define XMR_MMT_BN 128u
#define XMR_MMT_BK 16u
#define XMR_MMT_VT 128u
#define XMR_MMT_SMEM (64u * 1024u)
XMR_GEOM_FN unsigned xmr_mmt_threads(unsigned nc) { return nc * XMR_MMT_VT; }

/* ---- wgmma kernels (TF32 GEMM and the u8 limb matmul): warpgroup 0 produces, 1-2 consume; 128-row tiles; operand stages,
 * 1 KiB of alignment slack and 256 bytes of barriers ---- */
#define XMR_WG_THREADS      384
#define XMR_WG_BM           128u
#define XMR_WG_SMEM_TAIL    (1024u + 256u)
#define XMR_PREPASS_THREADS 256              /* the operand transposes and limb splits that run first */
/* TF32: BK = 32 fp32 (one 128-byte swizzle row); wide = 128 x 256 tiles (unprotected, N % 256 == 0), else 128 x 128 */
#define XMR_GEMM_BK 32u
XMR_GEOM_FN unsigned xmr_gemm_bn(int wide) { return wide ? 256u : 128u; }
XMR_GEOM_FN unsigned xmr_gemm_stages(int wide) { return wide ? 4u : 6u; }
XMR_GEOM_FN unsigned xmr_gemm_b_box(int pair) { return pair ? 64u : 128u; }   /* B^T rows per TMA box; a pair's CTAs load half each */
XMR_GEOM_FN unsigned xmr_gemm_smem(int wide) {
    return xmr_gemm_stages(wide) * (XMR_WG_BM * XMR_GEMM_BK * 4u + XMR_GEMM_BK * xmr_gemm_bn(wide) * 4u) + XMR_WG_SMEM_TAIL;
}
/* BF16: BK = 64 bf16 (the same 128-byte row, so the same stages and shared memory); B is read in place in boxes of 64 columns
 * (128 bytes, the widest row the 128-byte swizzle takes) x BK k-rows, for single CTAs and pairs alike */
#define XMR_GEMM_BF16_BK    64u
#define XMR_GEMM_BF16_B_BOX 64u
/* FP8 (E4M3): BK = 128 bytes, the same row again; B^T only (8-bit wgmma reads B K-major), in TF32's boxes of B^T rows */
#define XMR_GEMM_FP8_BK     128u
/* limbs: BK = 128 u8 of 4 planes, 2 stages; BN = 64 unprotected, 32 protected (register accumulators) */
#define XMR_MMTC_BK     128u
#define XMR_MMTC_STAGES 2u
XMR_GEOM_FN unsigned xmr_mmtc_bn(unsigned nc) { return nc == 1u ? 64u : 32u; }
XMR_GEOM_FN unsigned xmr_mmtc_smem(unsigned nc) {
    return XMR_MMTC_STAGES * (4u * XMR_WG_BM * XMR_MMTC_BK + 4u * xmr_mmtc_bn(nc) * XMR_MMTC_BK) + XMR_WG_SMEM_TAIL;
}

/* ---- quicksort: persistent warps, each with a private scratch slot ---- */
#define XMR_QSORT_THREADS 128

/* ---- ragged SHA-256 / CRC16 / quicksort (COAST_UNIT_OFFSETS): a counting-sort pre-pass orders the units by cost, longest
 * first, then a persistent grid pulls warp-tiles of consecutive permuted units from a counter (CTAs of XMR_CTA_THREADS for
 * SHA-256 and CRC16, XMR_QSORT_THREADS for quicksort).  Scratch layout:
 *   [0, 64)                 header: the offset table's address (u64) and the warp-tile counter (u32)
 *   [64, 64 + 4 * BUCKETS)  per-cost-bucket counts, then (after the scan) each bucket's next free slot
 *   [XMR_RAGGED_PERM, ..)   the permutation, one u32 unit index per unit
 *   quicksort only: from xmr_ragged_slots(n), 128-byte aligned, one slot of 32 x unit_bytes per warp of the grid (each lane
 *   group's NC x L copies sized by the bound, as in the uniform kernel)
 * Costs (XMR_RAGGED_COST_*): CRC16 bytes (0..255), SHA-256 compressions (nblk, the top bucket takes every nblk >= BUCKETS - 1),
 * quicksort elements (0..1024, the top bucket takes 1023 and 1024). */
#define XMR_RAGGED_BUCKETS      1024u
#define XMR_RAGGED_HDR          64u
#define XMR_RAGGED_PERM         (XMR_RAGGED_HDR + 4u * XMR_RAGGED_BUCKETS)
#define XMR_RAGGED_SCAN_THREADS 1024         /* the one-CTA scan: one thread per bucket */
#define XMR_RAGGED_COST_CRC     0u
#define XMR_RAGGED_COST_SHA     1u
#define XMR_RAGGED_COST_QSORT   2u
XMR_GEOM_FN unsigned long long xmr_ragged_scratch(unsigned long long n_units) { return XMR_RAGGED_PERM + 4ull * n_units; }
XMR_GEOM_FN unsigned long long xmr_ragged_slots(unsigned long long n_units) { return (xmr_ragged_scratch(n_units) + 127ull) & ~127ull; }

/* ---- grouped matmuls (COAST_MM_GROUPED, xmr_mm_grp.cuh): a group block in scratch = the rebased TF32 / BF16 / FP8 A tensor map (128 bytes),
 * then tile_start[G + 1] (u32), written by a one-CTA scan; at most XMR_MM_GRP_MAX groups per launch ---- */
#define XMR_MM_GRP_SCAN_THREADS 1024
#define XMR_MM_GRP_TILES        128u
#define XMR_MM_GRP_MAX          (1u << 20)
XMR_GEOM_FN unsigned long long xmr_mm_grp_bytes(unsigned long long groups) { return XMR_MM_GRP_TILES + 4ull * (groups + 1ull); }

#endif
