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
    COAST_K_COUNT_    = 8
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
 *   GEMM_TF32 same with float.
 *   QSORT    in : n_units x unit_bytes, arrays of L = unit_bytes/4 int32 (L <= 1024)   out: the sorted arrays
 *   CHSTONE_SHA in : n_units x unit_bytes stream bytes (unit_bytes a multiple of 64, 64 <= unit_bytes < 2^29)
 *            out: n_units x 5 uint32 = sha_info_digest[5] (sha.h:38)
 *   CHSTONE_AES in : n_units x 16 int32 = statemt[0..16) (aes.c:83; one byte per int, only the low 8 bits are used)
 *            out: n_units x 16 int32;  aux: n_units x 16 int32 keys with COAST_AES_KEY_PER_UNIT, else `key` below;
 *            mode bit0 = decrypt.  The key is never modified (KeySchedule expands into word[][], aes_key.c:129-163).
 */
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
    uint32_t M, N, K;      /* MM_U32 / GEMM_TF32                                  */
    const void* d_in;
    void*       d_out;
    const void* d_aux;
    uint8_t     key[16];   /* AES single-key mode                                 */
    const coast_fault_plan* plan; /* NULL = no injection                          */
    void*       d_status;  /* optional, n_units x uint8_t: per unit, the number of SoR-exit votes at which the
                              replicas disagreed (saturating at 255; 0 = all agreed).  This is the per-run "F:"
                              field of the board report line (decoder.py:66) for campaign tooling.  A device
                              pointer for coast_launch, a host pointer for coast_run_host (not for the matmuls). */
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
uint32_t coast_out_bytes(uint32_t kernel, uint32_t unit_bytes);          /* QSORT: unit_bytes, the sorted array */
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
 *   pinned buffers (cuMemHostAlloc, cudaHostAlloc/Register, coast_host_alloc, torch pin_memory)
 *     and a kernel that reads its input once (CRC16, SHA256, AES128, CHSTONE_SHA): ONE launch
 *     reads the mapped host memory through the TMA ring and writes the voted output straight
 *     back -- upload, compute and download overlap inside the kernel (zero-copy);
 *   anything else (pageable memory, matmuls, quicksort): staged -- H2D -> kernel -> D2H per
 *     chunk, chunks of 1..16 MiB round-robin over three internal streams and staging slots
 *     (a unit larger than 16 MiB is a chunk of its own).  d_status is staged per chunk too.
 * COAST_HOST_PATH=staged|zerocopy forces a path.  On any failure every copy already queued on
 * the caller's buffers is drained before the call returns. */
int  coast_run_host(const coast_launch_desc* desc_with_host_ptrs, coast_stats* out);
const char* coast_last_host_path(void);   /* "zerocopy", "staged" or "one-shot" (matmuls): what the last host call did */
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
