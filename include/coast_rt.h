/*
 * coast_rt.h -- C ABI of libcoast_rt.so, the H100 redundant-execution runtime.
 *
 * The reference (byuccl/coast) has NO run-time library: `opt -TMR/-DWC` inlines
 * replicas, voters and counters into the program.  The only run-time symbols it
 * leaves behind are
 *     i32  TMR_ERROR_CNT            projects/dataflowProtection/synchronization.cpp:38,269-291
 *     i64  __SYNC_COUNT             synchronization.cpp:47,103-121
 *     void FAULT_DETECTED_DWC(void) synchronization.cpp:36,1198-1267
 * This library exports exactly those three, plus a launch ABI that replaces
 *     dataflowProtection::run(M, numClones)   dataflowProtection.cpp:63-164
 *     TMR::runOnModule  -> run(M,3)           projects/TMR/TMR.cpp:29-36
 *     DWC::runOnModule  -> run(M,2)           projects/DWC/DWC.cpp:29-36
 * with a runtime "triplicate-and-vote" launch of a hand-written sm_90a kernel.
 *
 * Plain C, plain pointers and sizes.  No CUDA / torch types in any signature:
 * device pointers are `void*` (CUdeviceptr-compatible), streams are `void*`
 * (CUstream / cudaStream_t / torch's `cuda_stream` integer).  The library binds
 * to libcuda.so.1 lazily (dlopen) inside coast_init(), so it LOADS on a box
 * without a GPU and every compute entry point then fails loudly with
 * COAST_ERR_NO_DRIVER -- there is no CPU fallback in this library.
 *
 * Thread-safety: like the reference's emitted code (plain load/add/store on the
 * counters, synchronization.cpp:1428-1431) the host API is single-caller per
 * process: one counter block, one set of host-call staging slots.  It does not
 * race silently -- a second host thread that enters coast_init / coast_launch /
 * coast_sync* / coast_run_host* / coast_stats_* / coast_fill_philox / coast_shutdown
 * while a call is in progress gets COAST_ERR_BUSY.  Device counters are warp-reduced
 * and atomically added.
 */
#ifndef COAST_RT_H_
#define COAST_RT_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ */
/* Run-time symbols the reference pass creates/uses (same names/types) */
/* ------------------------------------------------------------------ */

/* synchronization.cpp:269-291 -- i32, zero-initialised, +1 per executed TMR sync
 * point at which any replica disagrees with r0 (when -countErrors is given).
 * Weak here: a test that defines its own (tests/pynq/matrixMultiply.tmr/mm_tmr.c:29)
 * wins at link time. */
extern uint32_t TMR_ERROR_CNT;
/* synchronization.cpp:103-121,1415-1425 -- i64, +1 per executed sync point
 * (-countSyncs; only emitted together with the TMR error counter). */
extern uint64_t __SYNC_COUNT;
/* synchronization.cpp:1198-1267 -- user-overridable DWC handler; the default the
 * pass synthesises calls abort() (:1251-1266).  Weak default here does the same. */
void FAULT_DETECTED_DWC(void);

/* ------------------------------------------------------------------ */
/* Protected workloads (SURVEY.md section 8a, rows a1-a8)              */
/* ------------------------------------------------------------------ */
typedef enum coast_kernel_id {
    COAST_K_CRC16     = 0, /* tests/crc16/crc16.c:21-31                        */
    COAST_K_SHA256    = 1, /* tests/sha256_common/sha256_common_tmr.c:28-180   */
    COAST_K_AES128    = 2, /* tests/aes/TI_aes_128.c:107-231                   */
    COAST_K_MM_U32    = 3, /* tests/mm_common/mm_common_tmr.c:3-20 (exact, mod 2^32;
                              same low 32 bits as matrixMultiply.c:95-112)      */
    COAST_K_GEMM_TF32 = 4, /* BASELINE config 4: fp32 in/out, wgmma tf32 */
    COAST_K_QSORT     = 5, /* tests/quicksort/quicksort.c:121-136 (SURVEY.md 8f-4): data-dependent branches -> the
                              branch conditions are the sync points, voted inside the loops */
    COAST_K_CHSTONE_SHA = 6, /* tests/chstone/sha/sha.c:93-193 (SURVEY.md 8f-4): the CHStone `sha` benchmark -- one unit
                                is one STREAM (a serial chain of unit_bytes/64 + 1 compressions), five u32 votes */
    COAST_K_CHSTONE_AES = 7, /* tests/chstone/aes/{aes_enc,aes_dec,aes_func,aes_key}.c (SURVEY.md 8f-4): CHStone `aes`, type 128128 --
                                one byte per int; 16 int votes */
    COAST_K_GEMM_BF16 = 8, /* bfloat16 in, fp32 accumulate and out, wgmma bf16; B is read in place (no pre-pass, no scratch) */
    /* 9 is not assigned: coast_launch refuses it as an unknown kernel */
    COAST_K_GEMM_FP8  = 10, /* FP8 E4M3 in, fp32 out, wgmma e4m3; B^T read K-major (a byte-transposing pre-pass without
                               COAST_MM_B_TRANSPOSED) */
    /* 11 is not assigned either */
    COAST_K_GEMM_I8   = 12, /* int8 (s8) in, int32 out, exact mod 2^32, wgmma s8; B^T read K-major as for GEMM_FP8; integer vote */
    /* 13 is not assigned either */
    COAST_K_GEMM_F16  = 14, /* float16 (IEEE binary16) in, fp32 accumulate and out (f16 with COAST_MM_OUT_F16), wgmma f16;
                               GEMM_BF16's layout: B read in place */
    COAST_K_COUNT_    = 15
} coast_kernel_id;

/* numClones of dataflowProtection::run: 3 = -TMR, 2 = -DWC, 1 = unprotected
 * single replica (the baseline the acceptance ratios are quoted against). */
#define COAST_UNPROTECTED 1u
#define COAST_DWC         2u
#define COAST_TMR         3u

/* OPT_PASSES tokens (dataflowProtection.cpp:14-47) that change the emitted code
 * on this path.  coast_parse_opt_passes() maps the token string onto these. */
#define COAST_F_COUNT_ERRORS        0x0001u /* -countErrors  synchronization.cpp:1354-1465 */
#define COAST_F_COUNT_SYNCS         0x0002u /* -countSyncs   synchronization.cpp:1415-1425 */
#define COAST_F_NO_MEM_REPLICATION  0x0004u /* -noMemReplication (rule D2, passes.rst "Replication Rules"): variables live ONCE, stores
                                               are voted (synchronization.cpp:205-215) -> in-loop store votes, see below */
#define COAST_F_INTERLEAVE          0x0008u /* -i : replicas on adjacent LANES of one warp (every kernel's native placement) */
#define COAST_F_SEGMENT             0x0010u /* -s : replicas on adjacent WARPS of one CTA (reference default,
                                               interface.cpp:245-247); layout hint only, results identical */
#define COAST_F_VERBOSE             0x0020u /* -verbose */
#define COAST_F_REPORT_ERRORS_LEGACY 0x0040u /* -reportErrors (deprecated; counts AGREEING syncs,
                                               synchronization.cpp:1323-1350).  Parsed, warned, NOT emulated. */
#define COAST_F_MAJORITY_VOTER      0x0100u /* extension: bitwise 2-of-3 majority instead of the reference's
                                               select voter.  Off by default (reference semantics). */
#define COAST_F_STORE_DATA_SYNC     0x0200u /* -storeDataSync: vote the data of every store (rule C4), synchronization.cpp:211-215 */
#define COAST_F_NO_STORE_DATA_SYNC  0x0400u /* -noStoreDataSync: no store-data votes (:333-335); the SoR-exit votes stay (:304-322) */
#define COAST_F_NO_LOAD_SYNC        0x0800u /* -noLoadSync: with -noMemReplication, no votes on load address offsets (C3, :347-360) */
#define COAST_F_NO_STORE_ADDR_SYNC  0x1000u /* -noStoreAddrSync: ... nor on store address offsets (C5, :362-375) */
/* IN-LOOP STORE VOTES = (-storeDataSync or -noMemReplication) and not -noStoreDataSync: every assignment to a data variable
 * of the protected function is voted and, under TMR, all replicas continue with the voted value; __SYNC_COUNT grows
 * accordingly (crc16: 3 per byte + 1; matrix_multiply: K + 1 per element; sha256: len + 720 per compression + 32).  Built for
 * CRC16, MM_U32 and SHA256 (which then run their general kernels).  The other kernels cannot honour it: they WARN on stderr and run the default sync set, or
 * fail with COAST_ERR_UNSUPPORTED when COAST_STRICT_FLAGS=1.  coast_flags_honoured() tells which.
 * Address-offset votes need a data-dependent subscript; crc16 and matrix_multiply have none, so -noLoadSync /
 * -noStoreAddrSync change nothing there (DESIGN.md). */

/* ------------------------------------------------------------------ */
/* Fault plan: the on-device replacement of simulation/platform         */
/* ------------------------------------------------------------------ */
/* Reference fault model: exactly one uniformly random single-bit flip
 * (`val ^ (1 << randint(0, bitlen-1))`, simulation/platform/resources/injector.py:202-207)
 * at a uniformly random location (:156-179) per run.  Here a "run" is one unit
 * (message / block / output element).  At most one flip per unit:
 *
 *   mode BERNOULLI: (x0,x1,x2,x3) = Philox4x32-10(ctr = {unit_lo, unit_hi, 0, 0},
 *                                                 key = {seed_lo, seed_hi})
 *        inject  iff x0 < threshold            (p = threshold / 2^32)
 *        replica = x1 % num_clones
 *        site    = x2 % n_sites(kernel, unit_bytes)   (coast_fault_sites())
 *        bit     = x3 % site_width_bits(kernel, site) (coast_fault_site_bits())
 *   mode TABLE: one u32 per unit on the device, COAST_FAULT_ENTRY(replica, site, bit)
 *        or 0 for "no fault" -- the analogue of `--forceBreak "set ADDR = VAL"`
 *        (supervisor.py:357-359).  Entries with replica >= num_clones, site >= n_sites
 *        or bit >= width are ignored (not counted as injected).
 *
 * `unit` is the GLOBAL unit index (coast_launch_desc.unit_base + local index) so a
 * sharded multi-GPU run sees the same fault distribution as a single-GPU run.
 * The enumerated sites (identical in oracle/ and in the kernels) are listed in
 * DESIGN.md section "Fault sites". */
#define COAST_PLAN_NONE      0u
#define COAST_PLAN_BERNOULLI 1u
#define COAST_PLAN_TABLE     2u
#define COAST_FAULT_ENTRY(replica, site, bit) \
    (0x80000000u | (((uint32_t)(replica) & 3u) << 29) | (((uint32_t)(site) & 0xFFFFFFu) << 5) | ((uint32_t)(bit) & 31u))

typedef struct coast_fault_plan {
    uint32_t mode;        /* COAST_PLAN_*                                   */
    uint32_t seed_lo;     /* Philox key word 0                               */
    uint32_t seed_hi;     /* Philox key word 1                               */
    uint32_t threshold;   /* BERNOULLI: inject iff x0 < threshold            */
    const void* d_table;  /* TABLE: device pointer, n_units x uint32_t       */
} coast_fault_plan;

/* ------------------------------------------------------------------ */
/* Launch descriptor                                                   */
/* ------------------------------------------------------------------ */
/* Layouts (all device pointers, caller-owned, dense, unit-major):
 *   CRC16    in : n_units x unit_bytes (1..255) message bytes   out: n_units x uint16_t
 *   SHA256   in : n_units x unit_bytes message bytes            out: n_units x 32 digest bytes
 *   AES128   in : n_units x 16 state bytes                      out: n_units x 16
 *            aux: per-unit 16-byte keys (n_units x 16) if COAST_AES_KEY_PER_UNIT in `mode`,
 *                 otherwise NULL and `key` below is the one ECB key.  mode bit0 = dir
 *                 (0 encrypt, 1 decrypt, as TI_aes_128.c:107's `dir`; the key passed is
 *                 always the ORIGINAL cipher key, :112-129).
 *   MM_U32   in : A, M x K uint32 row-major; aux: B, K x N uint32 row-major
 *            out: C, M x N uint32; a unit is one C element, n_units must be M*N.  Exact modulo 2^32 on every
 *            path: wgmma u8 x u8 on u8 limbs when M%128 == N%64 == K%128 == 0 (limb planes are per-launch scratch
 *            from a stream-ordered pool: any number of streams), register-tiled CUDA cores when M%64 == N%128 ==
 *            K%16 == 0, a plain kernel otherwise (e.g. the 9 x 9 tests).  COAST_MM_PATH=tc|tiled|naive overrides.
 *            With COAST_MM_BATCHED: `batch` products of one shape in one launch (see below).
 *            With COAST_MM_GROUPED: G products that share N and K, each with its own row count (see below).
 *   GEMM_TF32 same with float.
 *   GEMM_BF16 in : A, M x K bfloat16 row-major; aux: B, K x N bfloat16 row-major   out: C, M x N float: the fp32-accumulated
 *            sum of the exact bf16 x bf16 products.  M%128 == N%128 == K%64 == 0 (grouped: N and K only), buffers 16-byte
 *            aligned.  A unit is one C element with one fault site of width 32, as GEMM_TF32.  COAST_MM_BATCHED and
 *            COAST_MM_GROUPED as below; the element offsets there count 2-byte elements in d_in and d_aux, 4-byte ones in d_out
 *            (2-byte ones with COAST_MM_OUT_BF16: C is then bfloat16, see below).
 *   GEMM_FP8 in : A, M x K FP8 E4M3 row-major; aux: B, K x N FP8 E4M3 row-major   out: C, M x N float.  E4M3 is the OCP
 *            encoding of torch.float8_e4m3fn: no infinities, S.1111.111 is NaN.  The products are exact; they are summed in
 *            the tensor core's accumulator, whose width for FP8 is not fp32's (DESIGN.md §6), then written as fp32.
 *            M%128 == N%128 == K%128 == 0 (grouped: N and K only), buffers 16-byte aligned.  A unit is one C element with one
 *            fault site of width 32 and one fp32 vote, as GEMM_TF32.  The 8-bit wgmma reads B K-major only, so B is
 *            transposed into P*K*N bytes of scratch first; with COAST_MM_B_TRANSPOSED the caller's B^T is read in place.
 *            COAST_MM_BATCHED and COAST_MM_GROUPED as below; the element offsets count 1-byte elements in d_in and d_aux,
 *            4-byte ones in d_out (2-byte ones with COAST_MM_OUT_BF16).  With COAST_MM_SCALE_TENSOR or COAST_MM_SCALE_ROWWISE every replica multiplies its value
 *            by the scales of A and B before the vote (see below).
 *   GEMM_I8  in : A, M x K int8 row-major; aux: B, K x N int8 row-major   out: C, M x N int32:
 *            C[i][j] = sum_k a_ik * b_kj mod 2^32, as two's complement, for any K: the s32 accumulators have no .satfinite and
 *            wrap.  This equals MM_U32 on the sign-extended operands, and torch._int_mm whenever no sum leaves int32 (always for
 *            K < 2^17).  Shape and alignment rules, the B^T pre-pass and scratch, COAST_MM_BATCHED, COAST_MM_GROUPED and
 *            COAST_MM_B_TRANSPOSED are GEMM_FP8's (element offsets: 1-byte elements in d_in and d_aux, 4-byte ones in d_out).
 *            A unit is one C element with one fault site of width 32 (the s32 accumulator after the main loop) and one vote,
 *            GEMM_TF32's geometry, so a plan draws the faults of a GEMM_FP8 launch of the same shape.  The vote is INTEGER
 *            equality (`icmp eq`) with the select voter r0==r1 ? r0 : r2, or bitwise majority with COAST_F_MAJORITY_VOTER.
 *            The fp32 vote would be wrong on these words: a bit-31 flip of a zero C gives 0x80000000, which `fcmp oeq` takes
 *            for -0.0 == +0.0, so TMR's select voter would store INT_MIN silently and DWC would miss the flip; and every C in
 *            [-8388607, -1] or [2139095041, 2147483647] is a NaN pattern, which `fcmp oeq` would count as a disagreement.
 *            COAST_MM_SCALE_* and COAST_MM_OUT_BF16 are refused (COAST_ERR_BAD_ARG).
 *   GEMM_F16 in : A, M x K float16 (IEEE binary16) row-major; aux: B, K x N float16 row-major   out: C, M x N float: the
 *            fp32-accumulated sum of the exact f16 x f16 products (float16 with COAST_MM_OUT_F16, see below).  Every rule of
 *            GEMM_BF16 holds unchanged: M%128 == N%128 == K%64 == 0 (grouped: N and K only), buffers 16-byte aligned, B read in
 *            place MN-major with no pre-pass and no scratch, B^T (COAST_MM_B_TRANSPOSED) read in place K-major, COAST_MM_BATCHED
 *            and COAST_MM_GROUPED with element offsets counting 2-byte elements in d_in and d_aux, and the 2^31 bounds.  A unit is
 *            one C element with one fault site of width 32 on the accumulator and one `fcmp oeq` vote, as GEMM_TF32, so a plan
 *            draws the faults of a GEMM_BF16 launch of the same shape.  COAST_MM_SCALE_* and COAST_MM_OUT_BF16 are refused
 *            (COAST_ERR_BAD_ARG).
 *   MM_U32 / GEMM_TF32 / GEMM_BF16 / GEMM_FP8 / GEMM_I8 / GEMM_F16 with COAST_MM_B_TRANSPOSED: aux: B^T, N x K row-major per product (see below).
 *   QSORT    in : n_units x unit_bytes, arrays of L = unit_bytes/4 int32 (L <= 1024)   out: the sorted arrays
 *   CHSTONE_SHA in : n_units x unit_bytes stream bytes (unit_bytes a multiple of 64, 64 <= unit_bytes < 2^29)
 *            out: n_units x 5 uint32 = sha_info_digest[5] (sha.h:38)
 *   CHSTONE_AES in : n_units x 16 int32 = statemt[0..16) (aes.c:83; one byte per int, only the low 8 bits are used)
 *            out: n_units x 16 int32;  aux: n_units x 16 int32 keys with COAST_AES_KEY_PER_UNIT, else `key` below;
 *            mode bit0 = decrypt.  The key is never modified (KeySchedule expands into word[][], aes_key.c:129-163).
 *   CRC16 / SHA256 with COAST_UNIT_OFFSETS: in = the messages end to end, aux = n_units + 1 u64 byte offsets (see below).
 *   QSORT with COAST_UNIT_OFFSETS: in = int32 arrays end to end, aux = n_units + 1 u64 byte offsets (multiples of 4);
 *            out: each array sorted into the same byte range of d_out, d_out[off[u] .. off[u+1]); nothing else is written.
 */
/* Ragged batches (CRC16, SHA256 and QSORT only): with COAST_UNIT_OFFSETS in `mode`, the n_units units lie end to end in d_in
 * and d_aux points to n_units + 1 uint64_t byte offsets (8-byte aligned); unit u is d_in[off[u] .. off[u+1]).  unit_bytes is
 * then the caller's bound on every length: at most 255 for CRC16 (crc16.c:21 takes an unsigned char), at most 2^28 for
 * SHA256, a multiple of 4 in 4..4096 for QSORT; n_units must be below 2^32.  The launch equals n_units single-unit launches,
 * unit u with unit_bytes = its length, d_in + off[u] and unit_base + u: the same outputs, d_status bytes, summed counters
 * and minimum first_fault_unit.  Fault sites count per unit (a zero-length CRC16 unit has none: never injected, output
 * 0xFFFF, one exit vote).  The kernel clamps each length to [0, unit_bytes] (a decreasing pair counts as 0); coast_run_host
 * rejects such tables.  A shard passes off + lo with the same d_in and unit_base = lo.  The units are ordered by cost in a
 * pre-pass so that long units do not leave the replica lanes of short ones idle.  Any other kernel fails with
 * COAST_ERR_BAD_ARG.
 * QSORT: the units are int32 arrays; d_in and d_out are 4-byte aligned and every offset is a multiple of 4 (the kernel rounds
 * an offset down to one; coast_run_host rejects it).  Array u is sorted into d_out + off[u], the bytes it came from; bytes of
 * d_out outside [off[0], off[n_units]) are never written.  Fault sites are 33 L_u per array (width 32).  A zero-length array
 * (which the uniform launch refuses) has no sites, writes nothing, has d_status 0 and executes one sync point, the
 * `if (len < 2) return;` of quicksort.c:122.  A shard passes off + lo with the same d_in, the SAME d_out (unlike CRC16 and
 * SHA256, whose d_out is indexed by the shard's own units) and unit_base = lo.  COAST_QSORT_PATH=nested gives
 * COAST_ERR_UNSUPPORTED: a ragged batch runs the state-machine scheduling only. */
#define COAST_UNIT_OFFSETS      0x10000u
/* Batched matmuls (MM_U32, GEMM_TF32, GEMM_BF16, GEMM_FP8, GEMM_I8 and GEMM_F16 only): with COAST_MM_BATCHED in `mode`, M, N and K are the shape of ONE product and
 * n_units = batch x M x N.  d_in holds `batch` A matrices (M x K) end to end, d_aux `batch` B matrices (K x N) and d_out
 * receives `batch` C matrices (M x N), all dense and row-major.  The launch equals `batch` single launches, matrix b with
 * d_in + b*M*K, d_aux + b*K*N, d_out + b*M*N (elements) and unit_base + b*M*N: the same output bytes, summed counters and
 * minimum first_fault_unit.  Fault plans stay keyed by the global unit index (a TABLE plan has n_units entries), and the
 * in-loop store votes keep their meaning (K + 1 votes per unit on the plain kernel).  Each path's shape rules apply to the
 * per-matrix M, N and K; a TF32 / BF16 / FP8 / I8 / F16 CTA pair needs the per-matrix M to be a multiple of 256.  COAST_ERR_BAD_ARG for the bit on
 * any other kernel, for n_units zero or not a multiple of M*N, and for batch*M or batch*N (GEMM_BF16 and GEMM_F16 without COAST_MM_B_TRANSPOSED:
 * batch*K) at or above 2^31.  Without the
 * bit n_units must be M*N; with batch = 1 the launch is identical to an unbatched one.  A shard takes whole matrices
 * [b_lo, b_hi): the three pointers and unit_base offset as above, n_units = (b_hi - b_lo) x M x N. */
#define COAST_MM_BATCHED        0x20000u
/* Grouped matmuls (MM_U32, GEMM_TF32, GEMM_BF16, GEMM_FP8, GEMM_I8 and GEMM_F16 only): with COAST_MM_GROUPED in `mode`, M is the number of products G (at least 1) and N
 * and K are shared by all of them.  d_rows points to G + 1 non-decreasing uint64_t row offsets ro[] (8-byte aligned; a device
 * pointer for coast_launch, a host pointer for coast_run_host): product g has M_g = ro[g+1] - ro[g] rows (zero is allowed),
 * its A at d_in + ro[g]*K, its B at d_aux + g*K*N and its C at d_out + ro[g]*N (elements); d_aux holds the G dense K x N
 * matrices end to end.  n_units = R*N with R = ro[G] - ro[0] the rows of all products.  The launch equals G single launches,
 * product g with M = M_g and unit_base + (ro[g] - ro[0])*N: the same output elements, summed counters, minimum
 * first_fault_unit and d_status bytes (coast_launch).  Fault plans stay keyed by the global unit index (a TABLE plan has n_units
 * entries); the sites are those of the kernel (K for MM_U32, 1 for GEMM_TF32, GEMM_BF16, GEMM_FP8, GEMM_I8 and GEMM_F16) and the in-loop store votes keep K + 1 votes per
 * unit.  Each path's shape rules apply to N and K only: every M_g is allowed on every path.  The kernels clamp every offset to
 * [ro[0], ro[0] + R] and count a decreasing pair as zero rows, so a malformed table never reads or writes outside
 * [ro[0], ro[0] + R) rows of the buffers; coast_run_host (and Runtime.run) refuse a table that decreases or whose last offset is
 * not ro[0] + R.  COAST_ERR_BAD_ARG for the bit on any other kernel or with COAST_MM_BATCHED or COAST_UNIT_OFFSETS, for G = 0
 * or above 2^20, for n_units not a multiple of N, for R or G*N (GEMM_BF16 and GEMM_F16 without COAST_MM_B_TRANSPOSED: G*K) at or above 2^31,
 * and for a null or misaligned d_rows.  A shard
 * takes whole products [g_lo, g_hi): d_rows + g_lo with the same d_in and d_out, d_aux + g_lo*K*N, M = g_hi - g_lo,
 * n_units = (ro[g_hi] - ro[g_lo])*N and unit_base + (ro[g_lo] - ro[0])*N. */
#define COAST_MM_GROUPED        0x40000u
/* Transposed B (MM_U32, GEMM_TF32, GEMM_BF16, GEMM_FP8, GEMM_I8 and GEMM_F16 only), the layout of a linear layer's weight: with COAST_MM_B_TRANSPOSED in
 * `mode`, d_aux holds B^T, each product's B stored as N rows of K elements, row-major: element (k, n) of product p is at
 * d_aux[p*N*K + n*K + k].  It combines with COAST_MM_BATCHED and COAST_MM_GROUPED; the product offsets into d_aux (p*K*N
 * elements) and the shard rules stay as documented there.  The launch equals the same launch without the bit whose d_aux holds
 * every product's B = (B^T)^T: the same output bytes, summed counters, minimum first_fault_unit and d_status bytes.  Fault sites,
 * their widths, TABLE plans and the in-loop store votes are unchanged.  B^T is read in place: GEMM_TF32 runs no transposing
 * pre-pass and needs no B^T scratch, GEMM_BF16 and GEMM_F16 read B^T K-major, GEMM_FP8 and GEMM_I8 run no byte-transposing pre-pass and need no
 * scratch (a grouped launch still allocates its group block), MM_U32's limb path splits B^T like A.  Each path's shape
 * rules are unchanged; the 2^31 bound on B's stacked rows is on batch*N (grouped: G*N) for every kernel with the bit.
 * COAST_ERR_BAD_ARG for the bit on any other kernel. */
#define COAST_MM_B_TRANSPOSED   0x80000u
/* Scaled FP8 matmuls (GEMM_FP8 only), what torch._scaled_mm(a, b, scale_a, scale_b) computes with fp32 output.  One of two
 * bits; each combines with COAST_MM_BATCHED, COAST_MM_GROUPED and COAST_MM_B_TRANSPOSED:
 *   COAST_MM_SCALE_TENSOR : d_scale_a and d_scale_b each point to ONE float, applied to every element of every product;
 *   COAST_MM_SCALE_ROWWISE: d_scale_a holds one float per row of the stacked A, indexed like d_in's rows: M entries for one
 *     product, batch*M for a batch (product b row i at b*M + i), and for groups row r of d_in uses d_scale_a[r], so entries
 *     [ro[0], ro[G]) are read.  d_scale_b holds one float per column of each product's B, P*N entries (product p column n at
 *     p*N + n); with COAST_MM_B_TRANSPOSED column n of B is row n of B^T, so the indexing is the same.
 * Element (i, j) of replica r is v_r = (acc_r * sa_i) * sb_j, two fp32 multiplies rounded to nearest (tensorwise: sa_i = sa[0],
 * sb_j = sb[0], so a tensorwise launch equals a row-wise one with constant vectors, bit for bit).  The vote, the counters and
 * d_status work on v_0 .. v_{NC-1} as they do without scales on acc_r: the scale multiply is part of the protected function,
 * and what is voted is what is stored.  Every replica reads the one copy of a scale (-noMemReplication's load rule).
 * The fault site is unchanged: site 0 is the replica's final accumulator, 32 bits, flipped BEFORE the scale.  So a zero scale
 * hides a flip that leaves the accumulator finite (the unit counts as injected and no vote disagrees; inf or NaN times 0 is NaN,
 * which disagrees), a NaN scale makes every vote of its row or column disagree, and a multiply that rounds two different
 * accumulators to one value hides the flip as well.
 * d_scale_a and d_scale_b are device pointers for coast_launch and host pointers for coast_run_host, read only with a scale
 * bit.  COAST_ERR_BAD_ARG for a scale bit on any other kernel, for both bits together, for a null scale pointer, for d_scale_a
 * not 4-byte aligned and, row-wise, for d_scale_b not 8-byte aligned.  Shards: a row or product shard passes d_scale_a + its
 * first row and d_scale_b + p_lo*N; a grouped shard passes d_scale_a unchanged (its rows are absolute, like d_in's) and
 * d_scale_b + g_lo*N.  Tensorwise scales are passed unchanged. */
#define COAST_MM_SCALE_TENSOR   0x100000u
#define COAST_MM_SCALE_ROWWISE  0x200000u
/* BF16 output (GEMM_BF16 and GEMM_FP8 only): with COAST_MM_OUT_BF16 in `mode`, C is bfloat16.  It
 * combines with COAST_MM_BATCHED, COAST_MM_GROUPED and COAST_MM_B_TRANSPOSED.  C keeps its layout: row-major, the same element
 * offsets as above (d_out + b*M*N, d_out + ro[g]*N, ...), now counting 2-byte elements.  Element (i, j) of replica r is
 * x_r, the accumulator after the fault hook, rounded to bfloat16 to nearest even (cvt.rn; subnormals are kept, a NaN
 * becomes 0x7FFF): v_r = bf16(x_r).  The vote, `fcmp oeq` on the
 * widened values (+0 and -0 agree, NaN disagrees with everything), the select and majority voters (bitwise on the 16-bit
 * patterns), the counters and d_status work on v_0 .. v_{NC-1} as they do on x_r without the bit: the rounding is part of the
 * protected function, and what is voted is what is stored.  The fault sites are unchanged (one 32-bit site per element, on the
 * accumulator), so a plan draws the same faults as for the fp32-output launch.  A flip that the rounding absorbs counts in
 * `injected` but not in errors_corrected or dwc_detected, and leaves its d_status byte 0.  With at most one flip per unit (the
 * plans above), the bf16 C of any launch equals the fp32 C of the same launch and plan rounded to nearest even, for every NC,
 * voter and plan, except for the sign of a zero where TMR's select voter meets a sign flip on replica 0 of a value that rounds
 * to zero (DESIGN.md §3.13).  COAST_ERR_BAD_ARG for the bit on any other kernel; COAST_ERR_UNSUPPORTED with a scale bit
 * (scaled GEMM_FP8 writes fp32 C only, for now).  The alignment rules are unchanged.
 * coast_run_host stages and downloads C at 2 bytes per element.  coast_out_bytes() does not see the mode and returns the fp32
 * size (4); a caller sizes a bf16 C at 2 bytes per unit. */
#define COAST_MM_OUT_BF16       0x400000u
/* FP16 output (GEMM_F16 only): with COAST_MM_OUT_F16 in `mode`, C is float16 (IEEE binary16), what torch.matmul returns for
 * half tensors.  Everything COAST_MM_OUT_BF16 says above holds with f16 for bf16: the same layout and element offsets (2-byte
 * elements), the same fault sites, and each replica rounds its accumulator after the fault hook, v_r = f16(x_r), to nearest even
 * (cvt.rn.f16x2.f32: subnormals are kept, finite values of 65520 or more in magnitude become infinities, a NaN becomes 0x7FFF).
 * The vote (`fcmp oeq` on the widened values; the majority voter bitwise on the 16-bit patterns), the counters and d_status
 * work on the rounded values.  With at most one flip per unit, the f16 C equals the fp32 C of the same launch and plan rounded
 * to nearest even, except for the sign of a zero where TMR's select voter meets a sign flip on replica 0 of a value that rounds
 * to zero (DESIGN.md §3.15).  COAST_ERR_BAD_ARG for the bit on any other kernel and together with COAST_MM_OUT_BF16.
 * coast_run_host stages and downloads C at 2 bytes per element; coast_out_bytes() returns the fp32 size (4). */
#define COAST_MM_OUT_F16        0x800000u
#define COAST_AES_DECRYPT       0x1u
#define COAST_AES_KEY_PER_UNIT  0x2u
#define COAST_AES_KEY_WRITEBACK 0x4u   /* with KEY_PER_UNIT: store what aes_enc_dec() leaves in key[] (TI_aes_128.c:214-221 mutates
                                          it: the last round key after encrypt, the original key after decrypt) back into d_aux.
                                          key[] is replica memory that never crosses the SoR through a vote, so -- like unprotected
                                          code reading a protected global (verification.cpp:690-710) -- copy 0 is what is stored. */

typedef struct coast_launch_desc {
    uint32_t kernel;       /* coast_kernel_id                                    */
    uint32_t num_clones;   /* 1, 2 (DWC) or 3 (TMR)                               */
    uint32_t flags;        /* COAST_F_*                                           */
    uint32_t mode;         /* kernel-specific (AES: COAST_AES_*)                  */
    uint64_t n_units;      /* units in THIS launch                                */
    uint64_t unit_base;    /* global index of this launch's unit 0 (fault plans)  */
    uint32_t unit_bytes;   /* CRC16/SHA256: message length of every unit          */
    uint32_t M, N, K;      /* the matmuls (MM_U32, GEMM_TF32, GEMM_BF16, GEMM_FP8, GEMM_I8, GEMM_F16) */
    const void* d_in;
    void*       d_out;
    const void* d_aux;
    uint8_t     key[16];   /* AES single-key mode                                 */
    const coast_fault_plan* plan; /* NULL = no injection                          */
    void*       d_status;  /* optional, n_units x uint8_t: per unit, the number of SoR-exit votes at which the
                              replicas disagreed (saturating at 255; 0 = all agreed).  This is the per-run "F:"
                              field of the board report line (decoder.py:66) for campaign tooling.  A device
                              pointer for coast_launch, a host pointer for coast_run_host (not for the matmuls). */
    const void* d_rows;    /* COAST_MM_GROUPED only (read only with the bit): G + 1 u64 row offsets, see above */
    const void* d_scale_a; /* COAST_MM_SCALE_TENSOR / _ROWWISE only (read only with a bit): float scales of A's rows, see above */
    const void* d_scale_b; /* ... and of B's columns */
} coast_launch_desc;

/* Counters of everything launched since the last coast_sync(). */
typedef struct coast_stats {
    uint64_t errors_corrected; /* TMR: sync points with !(r0==r1 && r0==r2); needs COAST_F_COUNT_ERRORS */
    uint64_t dwc_detected;     /* DWC: units with >= 1 mismatching output element            */
    uint64_t syncs;            /* executed sync points; needs COAST_F_COUNT_SYNCS             */
    uint64_t injected;         /* units that received a flip                                  */
    uint64_t first_fault_unit; /* smallest global unit index with a disagreement, or UINT64_MAX */
} coast_stats;

/* Error codes (0 = ok).  Driver errors are returned as -(CUresult). */
#define COAST_OK              0
#define COAST_ERR_NO_DRIVER   (-100001) /* libcuda.so.1 / a CUDA device is not available      */
#define COAST_ERR_NOT_INIT    (-100002)
#define COAST_ERR_BAD_ARG     (-100003)
#define COAST_ERR_UNSUPPORTED (-100004)
#define COAST_ERR_BUSY        (-100005) /* another host thread is inside the library (single caller, see Thread-safety) */

/* --- lifetime ------------------------------------------------------ */
int  coast_init(int device);          /* bind libcuda, retain device's primary context, load the sm_90a module; moves the
                                         calling thread onto the CPUs of the GPU's NUMA node and prefers that node for its
                                         memory (the host-call path is PCIe-bound); COAST_NUMA_BIND=0 disables that */
int  coast_numa_node(void);           /* the node coast_init bound to, or -1 */
int  coast_shutdown(void);
const char* coast_last_error(void);   /* human-readable text of the last failure */
const char* coast_version(void);

/* --- the pass front end: OPT_PASSES string -> (num_clones, flags) -- */
/* Accepts the tokens of tests/<t>/Makefile OPT_PASSES (e.g. "-TMR -verbose -countErrors").
 * Unknown tokens are warned about on stderr and ignored, as `opt` would for passes
 * that are not loaded.  Returns 0, or COAST_ERR_BAD_ARG if both -TMR and -DWC. */
int  coast_parse_opt_passes(const char* opt_passes, uint32_t* num_clones, uint32_t* flags);
/* The subset of `flags` that changes what `kernel` executes (sync set, counters, replica layout); the rest is accepted
 * with a warning (or refused under COAST_STRICT_FLAGS=1). */
uint32_t coast_flags_honoured(uint32_t kernel, uint32_t num_clones, uint32_t flags);

/* --- the launch (replaces dataflowProtection::run + the emitted code) */
int  coast_launch(const coast_launch_desc* desc, void* stream);

/* Wait for `stream`, fold the device counters into *out (may be NULL) and into the
 * reference's globals: TMR_ERROR_CNT += errors_corrected (mod 2^32), __SYNC_COUNT += syncs;
 * then, if dwc_detected > 0, call FAULT_DETECTED_DWC() once (synchronization.cpp:1299-1302;
 * deferred to kernel completion -- a grid cannot abort() mid-flight).  Resets the device counters. */
int  coast_sync(void* stream, coast_stats* out);
/* Same, but never calls FAULT_DETECTED_DWC (campaign tooling wants the count, not SIGABRT). */
int  coast_sync_noabort(void* stream, coast_stats* out);
/* Copy the device counters into *out asynchronously-safe form without resetting/aborting.
 * `d_stats_out` variant: enqueue a D2D copy of the 5 counters (5 x u64) on `stream`, for
 * callers that all-reduce them across GPUs (NCCL) before looking at them. */
int  coast_stats_snapshot(void* stream, void* d_stats_out /* 5 x uint64_t on device */);

/* Measurement helpers (bench.py): number of SMs of the device, and one {clock64(), %globaltimer ns} record per SM written to
 * d_out[2 * smid], d_out[2 * smid + 1] (2 x uint64_t x coast_sm_count()).  Two probes around a timed region give the average SM
 * clock the region really ran at; NVML keeps reporting the nominal clock while tensor kernels run below it under the power limit. */
int  coast_sm_count(void);
int  coast_clock_probe(void* d_out, void* stream);

/* Multi-GPU fold of the counters inside the kernels, over NVLink peer memory, instead of a collective (SURVEY.md 8e: the
 * only exchange of the sharded path is the 40-byte counter block).  One process per GPU:
 *   owner  : coast_counters_export(handle)         -> 64 opaque bytes (a CUDA IPC handle of its counter block); ship them
 *            to the other ranks any way you like (a file, a pipe, torch.distributed);
 *   others : coast_counters_attach(handle)         -> every later kernel of this process adds its TMR_ERROR_CNT /
 *            __SYNC_COUNT / DWC / injected tallies (and min-folds first_fault_unit) into the OWNER's block with
 *            system-scope atomics; coast_sync() here waits for the stream and reports zeros, coast_stats_reset() is the
 *            owner's business;
 *   owner  : coast_sync() AFTER the others' streams have drained (a barrier of the caller's) reads the sum over all GPUs,
 *            folds it into TMR_ERROR_CNT / __SYNC_COUNT and calls FAULT_DETECTED_DWC() if any GPU saw a DWC mismatch.
 * Needs peer access between the GPUs (NVLink/NVSwitch or PCIe P2P); attach fails loudly otherwise. */
#define COAST_COUNTERS_HANDLE_BYTES 64
int  coast_counters_export(void* handle /* COAST_COUNTERS_HANDLE_BYTES */);
int  coast_counters_attach(const void* handle);
int  coast_counters_detach(void);
int  coast_stats_reset(void* stream);

/* --- fault-site geometry (shared by oracle and kernels) ------------- */
uint32_t coast_fault_sites(uint32_t kernel, uint32_t unit_bytes, uint32_t K);
uint32_t coast_fault_site_bits(uint32_t kernel, uint32_t unit_bytes, uint32_t K, uint32_t site);
uint32_t coast_out_bytes_per_unit(uint32_t kernel);                      /* 0 for QSORT (variable) */
uint32_t coast_out_bytes(uint32_t kernel, uint32_t unit_bytes);          /* QSORT: unit_bytes, the sorted array; the matmuls:
                                                                            the fp32 C size, 4 (COAST_MM_OUT_BF16 C: 2) */
uint32_t coast_votes_per_unit(uint32_t kernel);  /* sync points per unit at the SoR exit */

/* --- thin memory helpers for pure-C callers (no torch) --------------- */
int  coast_malloc(void** d_ptr, size_t bytes);
int  coast_free(void* d_ptr);
int  coast_memcpy_h2d(void* d_dst, const void* h_src, size_t bytes, void* stream);
int  coast_memcpy_d2h(void* h_dst, const void* d_src, size_t bytes, void* stream);
int  coast_memset(void* d_dst, int byte, size_t bytes, void* stream);
int  coast_host_alloc(void** h_ptr, size_t bytes);   /* pinned */
int  coast_host_free(void* h_ptr);
int  coast_stream_create(void** stream);
int  coast_stream_destroy(void* stream);
int  coast_stream_sync(void* stream);

/* Deterministic synthetic input: dst[i] (u32) = Philox4x32-10(ctr={i/4 (+word_base/4), 0,0,0}, key={seed,0})[i%4].
 * Same generator in oracle/ so CPU and GPU see identical bytes (SURVEY.md 8d). */
int  coast_fill_philox(void* d_dst, uint64_t n_words, uint64_t word_base, uint32_t seed, void* stream);

/* --- host-buffer convenience: the reference-facing call -------------- */
/* What the reference's protected function call becomes: host in -> xMR kernel -> host out,
 * counters folded as coast_sync().  d_in / d_out / d_aux / d_status of the descriptor are HOST
 * pointers here.
 *   staged (the default): H2D -> kernel -> D2H per chunk, chunks round-robin over three
 *     internal streams and staging slots, every slot reserved before the first copy.  Uniform
 *     units come in chunks of 1..16 MiB of input (COAST_HOST_CHUNK_BYTES; a unit larger than
 *     that is a chunk of its own); d_status is staged per chunk too;
 *   zerocopy: pinned buffers (cuMemHostAlloc, cudaHostAlloc/Register, coast_host_alloc, torch
 *     pin_memory) and a kernel that reads its input once (CRC16, SHA256, AES128, CHSTONE_SHA):
 *     ONE launch reads the mapped host memory and writes the voted output straight back; the
 *     default when the output is at most 1/8 of the input (CRC16, CHSTONE_SHA);
 *   hybrid: the staged chunks' kernels read a pinned input in place, outputs are staged;
 *   matmuls (MM_U32, GEMM_TF32, GEMM_BF16, GEMM_FP8, GEMM_I8, GEMM_F16): B goes up once and C comes down in row blocks (one-shot: one
 *     block for small or oddly shaped problems).
 * COAST_HOST_PATH=staged|hybrid|zerocopy forces a path, and for matmuls one-shot forces one block
 * (INTEGRATION.md §config).  Ragged calls (COAST_UNIT_OFFSETS, d_aux = host offsets, which must never
 * decrease nor give a length above unit_bytes, and for QSORT must be multiples of 4) are always staged: chunks are contiguous
 * unit ranges, each uploads its bytes and its slice of the offsets unchanged (QSORT also downloads the same byte range to
 * d_out + off[first]); a forced zerocopy or hybrid path gives COAST_ERR_UNSUPPORTED.  Batched matmuls (COAST_MM_BATCHED) are
 * staged in chunks of whole matrices sized by COAST_HOST_CHUNK_BYTES (a matrix larger than that is a chunk of its own): each
 * chunk uploads its A and B matrices, launches with its unit_base and downloads its C matrices.  Grouped matmuls
 * (COAST_MM_GROUPED) are staged in chunks of whole products whose A rows, B matrices, C rows and offsets fit COAST_HOST_CHUNK_BYTES
 * (a larger product is a chunk of its own): each uploads its slice of the offsets unchanged and launches with d_in and d_out
 * biased by ro[first] rows.  Scaled GEMM_FP8 (COAST_MM_SCALE_*) keeps the chunks of the unscaled call: tensorwise, the two
 * floats go up once; row-wise, row blocks send B's column scales once with B and each block its rows' A scales, batched chunks
 * the A rows and B columns of their products, grouped chunks A scales [ro[first], ro[end]) biased like d_in and B scales
 * [first*N, end*N).  With COAST_MM_OUT_BF16 or COAST_MM_OUT_F16 the same schedules move C at 2 bytes per element.  On any failure every copy already queued on
 * the caller's buffers is drained before the call returns. */
int  coast_run_host(const coast_launch_desc* desc_with_host_ptrs, coast_stats* out);
/* What the last host call did: "staged", "hybrid" or "zerocopy"; unbatched matmuls: "row-blocks" or "one-shot"; grouped: "groups". */
const char* coast_last_host_path(void);
/* Same, but never calls FAULT_DETECTED_DWC (fault campaigns want the count, not SIGABRT). */
int  coast_run_host_noabort(const coast_launch_desc* desc_with_host_ptrs, coast_stats* out);

/* The four reference entry points, callable from the UNCHANGED tests (the BOARD=b200
 * make flow redirects their calls here; INTEGRATION.md).  Protection mode comes from
 * coast_set_opt_passes() or the COAST_OPT_PASSES environment variable. */
int  coast_set_opt_passes(const char* opt_passes);
unsigned short coast_xmr_crc16(const unsigned char* data_p, unsigned char length);   /* crc16.c:21 */
void coast_xmr_sha256_hash(unsigned char ctx_data[], uint32_t ctx_bitlen[], uint32_t ctx_state[],
                           unsigned char data[], uint32_t len, unsigned char hash[]);   /* sha256_common_tmr.c:101 */
void coast_xmr_aes_enc_dec(unsigned char* state, unsigned char* key, unsigned char dir); /* TI_aes_128.c:107 */
void coast_xmr_matrix_multiply_u32(const uint32_t* f, const uint32_t* s, uint32_t* r, int side); /* mm_common_tmr.c:3 */
/* chstone/sha/sha.c:182-193 sha_stream(): hashes the vsize chunks indata[j][0 .. in_i[j]) (rows block_size bytes apart)
 * into digest[5].  The benchmark's globals are passed in by the generated glue; chunks must be multiples of 64 bytes. */
void coast_xmr_chstone_sha_stream(const unsigned char* indata, const int* in_i, int vsize, int block_size, uint32_t* digest);
/* chstone/aes: the cipher of encrypt() (dir 0, aes_enc.c:102-125) / decrypt() (dir 1, aes_dec.c:87-125) on statemt[], in place;
 * `type` must be 128128 (the benchmark's).  The printf and the main_result self-check of those functions are host effects
 * the generated glue reproduces. */
void coast_xmr_chstone_aes(int* statemt, const int* key, int type, int dir);

#ifdef __cplusplus
}
#endif
#endif /* COAST_RT_H_ */
