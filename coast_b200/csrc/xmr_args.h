/*
 * xmr_args.h -- kernel argument block shared by the host runtime (coast_rt.c, plain C)
 * and the sm_90a kernels (coast_kernels.cu).  Plain C layout, no CUDA types.
 */
#ifndef XMR_ARGS_H_
#define XMR_ARGS_H_

typedef struct xmr_args {
    const void* in;
    void* out;
    const void* aux;
    unsigned long long n_units;
    unsigned long long unit_base;
    unsigned long long* counters;     /* XMR_CTR_* slots, device memory            */
    const unsigned int* plan_table;   /* COAST_PLAN_TABLE: one u32 per local unit  */
    unsigned char* status;            /* optional: per-unit count of disagreeing votes (saturating u8) */
    unsigned int unit_bytes;
    unsigned int flags;               /* COAST_F_*                                  */
    unsigned int mode;                /* per kernel: AES, COAST_AES_* and the row pack (XMR_MODE_AES_ROWPACK_*); TF32 GEMM, XMR_MODE_* */
    unsigned int M, N, K;
    unsigned int plan_mode, seed_lo, seed_hi, threshold;
    unsigned int n_sites;
    unsigned int n_tiles;             /* TMA-tiled kernels: ceil(n_units / units-per-tile) */
    unsigned char key[16];
} xmr_args;

/* internal flag (set by the host in xmr_args.flags, never by callers): in-loop store votes are in effect (coast_rt.h) */
#define XMR_F_STORE_VOTES 0x8000u
/* AES: bits 8..11 of xmr_args.mode = log2 of the blocks per tensor-map row (the host describes the dense 16-byte blocks as
 * 64- or 256-byte rows when the count allows) */
#define XMR_MODE_AES_ROWPACK_SHIFT 8
#define XMR_MODE_AES_ROWPACK_MASK  0xFu
/* TF32 GEMM (set by the host from COAST_GEMM_*): tile-rows per rasterisation group (0 = the kernel's default), L2 eviction
 * hints on, no splitting of a short last round's tiles */
#define XMR_MODE_GROUP_M_MASK  0xFFu
#define XMR_MODE_L2_HINTS      0x100u
#define XMR_MODE_NO_TAIL_SPLIT 0x200u
/* scaled FP8 GEMM (xmr_scaled_fp8*; the host sets it for COAST_MM_SCALE_ROWWISE): one A scale per row and one B scale per
 * column of each product, instead of one of each */
#define XMR_MODE_SCALE_ROWWISE 0x400u

/* counter slots (mirror coast_stats) */
#define XMR_CTR_ERRORS   0
#define XMR_CTR_DWC      1
#define XMR_CTR_SYNCS    2
#define XMR_CTR_INJECTED 3
#define XMR_CTR_FIRST    4
#define XMR_CTR_COUNT    5

#endif
