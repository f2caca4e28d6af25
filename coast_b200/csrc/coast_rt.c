/*
 * coast_rt.c -- host side of libcoast_rt.so (plain C over the CUDA DRIVER API).
 *
 * Replaces, at run time, what byuccl/coast does at compile time:
 *   projects/dataflowProtection (run(M, numClones), dataflowProtection.cpp:63-164),
 *   projects/TMR (TMR.cpp:29-36) and projects/DWC (DWC.cpp:29-36)
 * by launching a hand-written sm_90a kernel in which every live value of the protected
 * region is computed by num_clones replicas and voted at the SoR exit.
 *
 * libcuda.so.1 is bound lazily with dlopen() so that this library LOADS without a GPU
 * (the CPU CI box) -- every compute entry point then returns COAST_ERR_NO_DRIVER.  There
 * is deliberately NO CPU implementation of the workloads in this file.
 */
#define _GNU_SOURCE
#include "../../include/coast_rt.h"
#include "xmr_args.h"
#include "xmr_geom.h"

#include <cuda.h>
#include <ctype.h>
#include <dlfcn.h>
#include <sched.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/syscall.h>
#include <unistd.h>

extern const unsigned char coast_kernels_cubin[];   /* generated: bin2c of coast_kernels.cubin */

/* ------------------------------------------------------------------ */
/* the reference's run-time symbols                                     */
/* ------------------------------------------------------------------ */
__attribute__((weak)) uint32_t TMR_ERROR_CNT = 0;    /* synchronization.cpp:269-291 */
__attribute__((weak)) uint64_t __SYNC_COUNT = 0;     /* synchronization.cpp:103-121 */
__attribute__((weak)) void FAULT_DETECTED_DWC(void) { /* synchronization.cpp:1251-1266: default handler = abort() */
    fprintf(stderr, "coast_rt: DWC mismatch detected -> FAULT_DETECTED_DWC -> abort()\n");
    abort();
}

/* ------------------------------------------------------------------ */
/* driver API binding                                                   */
/* ------------------------------------------------------------------ */
#define DRV_FUNCS(X)                                                                                         \
    X(cuInit, (unsigned int))                                                                                \
    X(cuDeviceGet, (CUdevice*, int))                                                                         \
    X(cuDeviceGetAttribute, (int*, CUdevice_attribute, CUdevice))                                            \
    X(cuDeviceGetPCIBusId, (char*, int, CUdevice))                                                           \
    X(cuPointerGetAttribute, (void*, CUpointer_attribute, CUdeviceptr))                                      \
    X(cuDevicePrimaryCtxRetain, (CUcontext*, CUdevice))                                                      \
    X(cuDevicePrimaryCtxRelease_v2, (CUdevice))                                                              \
    X(cuCtxSetCurrent, (CUcontext))                                                                          \
    X(cuCtxGetCurrent, (CUcontext*))                                                                         \
    X(cuModuleLoadData, (CUmodule*, const void*))                                                            \
    X(cuModuleUnload, (CUmodule))                                                                            \
    X(cuModuleGetFunction, (CUfunction*, CUmodule, const char*))                                             \
    X(cuFuncSetAttribute, (CUfunction, CUfunction_attribute, int))                                           \
    X(cuOccupancyMaxActiveBlocksPerMultiprocessor, (int*, CUfunction, int, size_t))                          \
    X(cuLaunchKernel, (CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned,     \
                       CUstream, void**, void**))                                                            \
    X(cuMemAlloc_v2, (CUdeviceptr*, size_t))                                                                 \
    X(cuMemFree_v2, (CUdeviceptr))                                                                           \
    X(cuMemPoolCreate, (CUmemoryPool*, const CUmemPoolProps*))                                               \
    X(cuMemPoolDestroy, (CUmemoryPool))                                                                      \
    X(cuMemPoolSetAttribute, (CUmemoryPool, CUmemPool_attribute, void*))                                     \
    X(cuMemAllocFromPoolAsync, (CUdeviceptr*, size_t, CUmemoryPool, CUstream))                               \
    X(cuMemFreeAsync, (CUdeviceptr, CUstream))                                                               \
    X(cuMemcpyHtoDAsync_v2, (CUdeviceptr, const void*, size_t, CUstream))                                    \
    X(cuMemcpyDtoHAsync_v2, (void*, CUdeviceptr, size_t, CUstream))                                          \
    X(cuMemcpyDtoDAsync_v2, (CUdeviceptr, CUdeviceptr, size_t, CUstream))                                    \
    X(cuMemsetD8Async, (CUdeviceptr, unsigned char, size_t, CUstream))                                       \
    X(cuMemHostAlloc, (void**, size_t, unsigned int))                                                        \
    X(cuMemFreeHost, (void*))                                                                                \
    X(cuStreamCreate, (CUstream*, unsigned int))                                                             \
    X(cuStreamDestroy_v2, (CUstream))                                                                        \
    X(cuStreamSynchronize, (CUstream))                                                                       \
    X(cuEventCreate, (CUevent*, unsigned int))                                                               \
    X(cuEventRecord, (CUevent, CUstream))                                                                    \
    X(cuEventDestroy_v2, (CUevent))                                                                          \
    X(cuStreamWaitEvent, (CUstream, CUevent, unsigned int))                                                  \
    X(cuGetErrorString, (CUresult, const char**))                                                            \
    X(cuIpcGetMemHandle, (CUipcMemHandle*, CUdeviceptr))                                                     \
    X(cuIpcOpenMemHandle_v2, (CUdeviceptr*, CUipcMemHandle, unsigned int))                                   \
    X(cuIpcCloseMemHandle, (CUdeviceptr))                                                                    \
    X(cuTensorMapEncodeTiled, (CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,      \
                               const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, \
                               CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill))

#define X(name, args) static CUresult(CUDAAPI* p_##name) args;
DRV_FUNCS(X)
#undef X

/* A tiled tensor map as the launch wants it.  `base` is an offset into the launch's scratch when in_scratch is set.
 * No padding: the map cache compares descriptions with memcmp. */
typedef struct {
    uintptr_t base;
    cuuint64_t dim[3], stride[2];
    cuuint32_t box[3], rank;
    CUtensorMapDataType dtype;
    CUtensorMapSwizzle swz;
    CUtensorMapL2promotion l2;
    int in_scratch;
} map_desc;
_Static_assert(sizeof(map_desc) == 80, "map_desc has no padding");

/* coast_run_host staging: a device buffer and its capacity; a slot is one host-call stream and the buffers its chunks use */
typedef struct { CUdeviceptr p; size_t cap; } dev_buf;
typedef struct { CUstream s; dev_buf in, out, aux, stat, rows, sc; } host_slot;   /* sc: a chunk's scales, A's then B's */

#define MAX_FN 128
static struct {
    int inited;
    void* libcuda;
    int device;
    CUdevice dev;
    CUcontext ctx;
    CUmodule mod;
    int sm_count;
    CUdeviceptr counters;            /* XMR_CTR_COUNT x u64 */
    CUdeviceptr peer_counters;       /* coast_counters_attach(): ANOTHER GPU's counter block, mapped over NVLink (0: not attached) */
    uint64_t* h_counters;            /* pinned mirror */
    struct { char name[64]; CUfunction fn; int ctas_per_sm; unsigned smem; } fns[MAX_FN];
    int n_fns;
    char err[512];
    /* protection mode of the four reference entry points (coast_set_opt_passes / COAST_OPT_PASSES) */
    uint32_t def_nc, def_flags; int def_set;
    host_slot slot[3];               /* coast_run_host: chunk i runs on slot i % 3 */
    dev_buf h_b; CUevent ev_b;       /* matmul host call: the replicated operand B (and the scales every chunk shares) and "B has landed" */
    /* stream-ordered scratch (the replicas' private arrays of xmr_qsort.cuh): any number of streams may launch at once */
    CUmemoryPool pool;
    int numa_node;                   /* NUMA node the process was bound to by coast_init (-1: not bound) */
    int busy;                        /* one host thread at a time (the reference is single-threaded); others fail loudly */
    /* tensor maps of the row-tiled kernels: coast_run_host re-encodes the same few maps every call */
    struct { map_desc key; CUtensorMap map; } tmaps[16];
    int n_tmaps, tmap_next;
    unsigned warned_store_votes;     /* one warning per kernel and process */
    int host_path_default;           /* host-call path for pinned buffers: 0 = staged, 1 = hybrid, 2 = zero-copy */
    const char* last_host_path;      /* "staged" | "hybrid" | "zerocopy" | "row-blocks" | "one-shot" | "groups": what the last coast_run_host did */
} G;

/* Single-caller guard.  The reference's emitted code is single-threaded (plain load/add/store on its counters,
 * synchronization.cpp:1428-1431) and so is this runtime: one counter block, one set of host-call slots.  A second host
 * thread entering while a call is in progress gets COAST_ERR_BUSY instead of a silent race. */
static int enter(void);
static void leave(void) { __atomic_store_n(&G.busy, 0, __ATOMIC_RELEASE); }

static int fail(int code, const char* fmt, ...) {
    va_list ap; va_start(ap, fmt);
    vsnprintf(G.err, sizeof G.err, fmt, ap);
    va_end(ap);
    return code;
}
static int enter(void) {
    if (__atomic_exchange_n(&G.busy, 1, __ATOMIC_ACQUIRE)) {
        /* do not touch G.err: the call in progress owns it */
        return COAST_ERR_BUSY;
    }
    return COAST_OK;
}
#define ENTER() do { int e_ = enter(); if (e_) return e_; } while (0)
#define LEAVE(rc) do { int l_ = (rc); leave(); return l_; } while (0)
static int drv_fail(CUresult r, const char* what) {
    const char* s = NULL;
    if (p_cuGetErrorString) p_cuGetErrorString(r, &s);
    return fail(-(int)r, "%s: CUDA error %d (%s)", what, (int)r, s ? s : "?");
}
#define DRV(call) do { CUresult r_ = (call); if (r_ != CUDA_SUCCESS) return drv_fail(r_, #call); } while (0)

const char* coast_last_error(void) { return G.err; }
const char* coast_version(void) { return "coast_rt 0.1 (sm_90a)"; }

static int bind_driver(void) {
    if (G.libcuda) return COAST_OK;
    void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libcuda.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return fail(COAST_ERR_NO_DRIVER, "libcuda.so.1 not found (%s): no GPU driver on this machine; "
                                              "libcoast_rt has no CPU fallback", dlerror());
#define X(name, args)                                                                 \
    *(void**)(&p_##name) = dlsym(h, #name);                                           \
    if (!p_##name) { dlclose(h); return fail(COAST_ERR_NO_DRIVER, "libcuda lacks %s", #name); }
    DRV_FUNCS(X)
#undef X
    G.libcuda = h;
    return COAST_OK;
}


/* ------------------------------------------------------------------ */
/* NUMA placement                                                        */
/* ------------------------------------------------------------------ */
/* The host-call path (coast_run_host) is PCIe-bound; on a two-socket box a process that runs -- and first-touches its
 * pinned buffers -- on the socket the GPU is NOT attached to can lose up to half of the copy
 * bandwidth.  coast_init() therefore moves the calling thread (threads it creates later inherit it) onto the CPUs of the GPU's NUMA node and makes that node the preferred one for its memory.  Plain syscalls, no
 * libnuma.  COAST_NUMA_BIND=0 leaves the process alone.  Best effort: any failure leaves things as they were. */
#ifndef MPOL_PREFERRED
#define MPOL_PREFERRED 1
#endif
static int parse_cpulist(const char* s, cpu_set_t* set) {
    int n = 0;
    CPU_ZERO(set);
    while (*s) {
        while (*s == ',' || isspace((unsigned char)*s)) ++s;
        if (!isdigit((unsigned char)*s)) break;
        char* e; long a = strtol(s, &e, 10), b = a;
        if (*e == '-') b = strtol(e + 1, &e, 10);
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int)c, set); ++n; }
        s = e;
    }
    return n;
}
static void numa_bind_to_gpu(void) {
    G.numa_node = -1;
    const char* env = getenv("COAST_NUMA_BIND");
    if (env && !strcmp(env, "0")) return;
    char bdf[32] = {0}, path[128], buf[4096];
    if (p_cuDeviceGetPCIBusId(bdf, (int)sizeof bdf - 1, G.dev) != CUDA_SUCCESS) return;
    for (char* c = bdf; *c; ++c) *c = (char)tolower((unsigned char)*c);
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bdf);
    FILE* f = fopen(path, "r"); if (!f) return;
    int node = -1; if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f);
    if (node < 0 || node >= 1024) return;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r"); if (!f) return;
    size_t got = fread(buf, 1, sizeof buf - 1, f); fclose(f); buf[got] = 0;
    cpu_set_t want, cur, both;
    if (!parse_cpulist(buf, &want)) return;
    if (sched_getaffinity(0, sizeof cur, &cur)) return;
    CPU_AND(&both, &want, &cur);                       /* never widen a cpuset the launcher (cgroup, taskset) imposed */
    if (!CPU_COUNT(&both)) return;
    if (sched_setaffinity(0, sizeof both, &both)) return;
    unsigned long mask[16]; memset(mask, 0, sizeof mask);
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    syscall(SYS_set_mempolicy, MPOL_PREFERRED, mask, (unsigned long)(8 * sizeof mask));   /* a refusal only costs locality */
    G.numa_node = node;
}
int coast_numa_node(void) { return G.inited ? G.numa_node : -1; }

static int ensure_ctx(void) {
    if (!G.inited) return fail(COAST_ERR_NOT_INIT, "coast_init() has not been called");
    CUcontext cur = NULL;
    p_cuCtxGetCurrent(&cur);
    if (cur != G.ctx) DRV(p_cuCtxSetCurrent(G.ctx));
    return COAST_OK;
}

static int get_fn(const char* name, unsigned smem, unsigned block, CUfunction* fn, int* ctas_per_sm) {
    for (int i = 0; i < G.n_fns; ++i)
        if (!strcmp(G.fns[i].name, name) && G.fns[i].smem == smem) { *fn = G.fns[i].fn; if (ctas_per_sm) *ctas_per_sm = G.fns[i].ctas_per_sm; return COAST_OK; }
    CUfunction f = NULL;
    CUresult r = p_cuModuleGetFunction(&f, G.mod, name);
    if (r != CUDA_SUCCESS) return drv_fail(r, name);
    if (smem > 48 * 1024) DRV(p_cuFuncSetAttribute(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem));
    int occ = 1;
    DRV(p_cuOccupancyMaxActiveBlocksPerMultiprocessor(&occ, f, (int)block, smem));
    if (occ < 1) occ = 1;
    if (G.n_fns < MAX_FN) {
        snprintf(G.fns[G.n_fns].name, sizeof G.fns[0].name, "%s", name);
        G.fns[G.n_fns].fn = f; G.fns[G.n_fns].ctas_per_sm = occ; G.fns[G.n_fns].smem = smem;
        G.n_fns++;
    }
    *fn = f; if (ctas_per_sm) *ctas_per_sm = occ;
    return COAST_OK;
}

static int launch_small(const char* name, unsigned grid, unsigned block, void** params, CUstream s) {
    CUfunction f; int rc = get_fn(name, 0, block, &f, NULL);
    if (rc) return rc;
    DRV(p_cuLaunchKernel(f, grid, 1, 1, block, 1, 1, 0, s, params, NULL));
    return COAST_OK;
}

static int stats_reset_impl(void* stream) {
    int rc = ensure_ctx(); if (rc) return rc;
    void* params[] = { &G.counters };
    return launch_small("xmr_counters_reset", 1, 32, params, (CUstream)stream);
}
int coast_stats_reset(void* stream) { ENTER(); LEAVE(stats_reset_impl(stream)); }

/* COAST_REPORT_COUNTERS=1: print the reference's two run-time symbols when the process exits -- what a debugger would read
 * out of a board (passes.rst "Error Logging"); the unchanged tests never print them */
static void report_counters(void) {
    fprintf(stderr, "coast_rt: TMR_ERROR_CNT=%u __SYNC_COUNT=%llu\n", TMR_ERROR_CNT, (unsigned long long)__SYNC_COUNT);
}

static int init_impl(int device) {
    if (G.inited) {
        if (device == G.device) return ensure_ctx();
        return fail(COAST_ERR_BAD_ARG, "coast_rt already initialised on device %d", G.device);
    }
    int rc = bind_driver(); if (rc) return rc;
    CUresult r = p_cuInit(0);
    if (r != CUDA_SUCCESS) { drv_fail(r, "cuInit"); return COAST_ERR_NO_DRIVER; }
    DRV(p_cuDeviceGet(&G.dev, device));
    DRV(p_cuDevicePrimaryCtxRetain(&G.ctx, G.dev));      /* shared with the CUDA runtime / torch */
    DRV(p_cuCtxSetCurrent(G.ctx));
    int major = 0, minor = 0;
    p_cuDeviceGetAttribute(&major, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR, G.dev);
    p_cuDeviceGetAttribute(&minor, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR, G.dev);
    if (major != 9 || minor != 0) {
        p_cuDevicePrimaryCtxRelease_v2(G.dev);
        return fail(COAST_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library carries sm_90a code only", device, major, minor);
    }
    p_cuDeviceGetAttribute(&G.sm_count, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, G.dev);
    numa_bind_to_gpu();
    G.host_path_default = 0;        /* staged: the copy engines move the bytes */
    r = p_cuModuleLoadData(&G.mod, coast_kernels_cubin);
    if (r != CUDA_SUCCESS) { p_cuDevicePrimaryCtxRelease_v2(G.dev); return drv_fail(r, "cuModuleLoadData(sm_90a cubin)"); }
    DRV(p_cuMemAlloc_v2(&G.counters, XMR_CTR_COUNT * sizeof(uint64_t)));
    {
        CUmemPoolProps pp; memset(&pp, 0, sizeof pp);
        pp.allocType = CU_MEM_ALLOCATION_TYPE_PINNED;
        pp.location.type = CU_MEM_LOCATION_TYPE_DEVICE; pp.location.id = (int)G.dev;
        DRV(p_cuMemPoolCreate(&G.pool, &pp));
        cuuint64_t keep = ~(cuuint64_t)0;                  /* keep freed scratch cached in the pool between launches */
        DRV(p_cuMemPoolSetAttribute(G.pool, CU_MEMPOOL_ATTR_RELEASE_THRESHOLD, &keep));
    }
    DRV(p_cuMemHostAlloc((void**)&G.h_counters, XMR_CTR_COUNT * sizeof(uint64_t), 0));
    G.device = device;
    G.inited = 1;
    rc = stats_reset_impl(NULL); if (rc) return rc;
    DRV(p_cuStreamSynchronize(NULL));
    const char* env = getenv("COAST_OPT_PASSES");
    if (env && !G.def_set) coast_set_opt_passes(env);
    { const char* rc_env = getenv("COAST_REPORT_COUNTERS"); static int registered;
      if (rc_env && strcmp(rc_env, "0") && !registered) { registered = 1; atexit(report_counters); } }
    return COAST_OK;
}
int coast_init(int device) { ENTER(); LEAVE(init_impl(device)); }

static int shutdown_impl(void) {
    if (!G.inited) return COAST_OK;
    ensure_ctx();
    dev_buf* bufs[] = { &G.h_b, &G.slot[0].in, &G.slot[0].out, &G.slot[0].aux, &G.slot[0].stat, &G.slot[0].rows, &G.slot[0].sc,
                        &G.slot[1].in, &G.slot[1].out, &G.slot[1].aux, &G.slot[1].stat, &G.slot[1].rows, &G.slot[1].sc,
                        &G.slot[2].in, &G.slot[2].out, &G.slot[2].aux, &G.slot[2].stat, &G.slot[2].rows, &G.slot[2].sc };
    for (size_t i = 0; i < sizeof bufs / sizeof bufs[0]; ++i) if (bufs[i]->p) p_cuMemFree_v2(bufs[i]->p);
    for (int i = 0; i < 3; ++i) if (G.slot[i].s) p_cuStreamDestroy_v2(G.slot[i].s);
    if (G.ev_b) p_cuEventDestroy_v2(G.ev_b);
    memset(G.slot, 0, sizeof G.slot); memset(&G.h_b, 0, sizeof G.h_b); G.ev_b = NULL;
    G.n_tmaps = G.tmap_next = 0;
    if (G.peer_counters) { p_cuIpcCloseMemHandle(G.peer_counters); G.peer_counters = 0; }
    p_cuMemFree_v2(G.counters);
    if (G.pool) { p_cuMemPoolDestroy(G.pool); G.pool = NULL; }
    p_cuMemFreeHost(G.h_counters);
    p_cuModuleUnload(G.mod);
    p_cuDevicePrimaryCtxRelease_v2(G.dev);
    G.inited = 0; G.n_fns = 0;
    return COAST_OK;
}
int coast_shutdown(void) { ENTER(); LEAVE(shutdown_impl()); }

/* ------------------------------------------------------------------ */
/* OPT_PASSES front end (dataflowProtection.cpp:14-47 cl::opt names)     */
/* ------------------------------------------------------------------ */
int coast_parse_opt_passes(const char* s, uint32_t* num_clones, uint32_t* flags) {
    uint32_t nc = COAST_UNPROTECTED, fl = 0; int tmr = 0, dwc = 0;
    if (!s) s = "";
    char buf[1024]; snprintf(buf, sizeof buf, "%s", s);
    for (char* tok = strtok(buf, " \t\r\n"); tok; tok = strtok(NULL, " \t\r\n")) {
        if (tok[0] == '#') break;                            /* rest of a Makefile line comment */
        if (!strcmp(tok, "-TMR")) tmr = 1;
        else if (!strcmp(tok, "-DWC")) dwc = 1;
        else if (!strcmp(tok, "-countErrors")) fl |= COAST_F_COUNT_ERRORS;
        else if (!strcmp(tok, "-countSyncs")) fl |= COAST_F_COUNT_SYNCS;
        else if (!strcmp(tok, "-noMemReplication")) fl |= COAST_F_NO_MEM_REPLICATION;
        else if (!strcmp(tok, "-storeDataSync")) fl |= COAST_F_STORE_DATA_SYNC;
        else if (!strcmp(tok, "-noStoreDataSync")) fl |= COAST_F_NO_STORE_DATA_SYNC;
        else if (!strcmp(tok, "-noLoadSync")) fl |= COAST_F_NO_LOAD_SYNC;
        else if (!strcmp(tok, "-noStoreAddrSync")) fl |= COAST_F_NO_STORE_ADDR_SYNC;
        else if (!strcmp(tok, "-i")) fl |= COAST_F_INTERLEAVE;
        else if (!strcmp(tok, "-s")) fl |= COAST_F_SEGMENT;
        else if (!strcmp(tok, "-verbose")) fl |= COAST_F_VERBOSE;
        else if (!strcmp(tok, "-reportErrors")) {
            fl |= COAST_F_REPORT_ERRORS_LEGACY;
            fprintf(stderr, "coast_rt: -reportErrors is deprecated in the reference (counts AGREEING syncs, "
                            "synchronization.cpp:1323-1350) and is not emulated; use -countErrors\n");
        }
        else fprintf(stderr, "coast_rt: OPT_PASSES token '%s' has no effect on the GPU runtime (ignored)\n", tok);
    }
    if (tmr && dwc) return fail(COAST_ERR_BAD_ARG, "-TMR and -DWC are mutually exclusive");
    if (tmr) nc = COAST_TMR; else if (dwc) nc = COAST_DWC;
    if (num_clones) *num_clones = nc;
    if (flags) *flags = fl;
    return COAST_OK;
}

/* ------------------------------------------------------------------ */
/* per-kernel facts                                                     */
/* ------------------------------------------------------------------ */
#define IN_UNIT_BYTES 0xFFFFFFFFu           /* kernel_info.in_bytes: the descriptor's unit_bytes */
static const struct kernel_info {
    const char* name;                       /* in messages */
    uint32_t out_bytes;                     /* per unit; QSORT: 0, the output is the unit's array */
    uint32_t votes;                         /* SoR-exit votes per unit */
    uint32_t in_bytes;                      /* per unit, staged by the host call; 0: the matmuls (operands, not units) */
    uint32_t key_bytes;                     /* per-unit key bytes with COAST_AES_KEY_PER_UNIT */
    int store_votes;                        /* in-loop store votes are built (coast_rt.h) */
    int streams_once;                       /* reads each input byte once: may read mapped host memory directly */
    uint32_t mm_elem;                       /* the matmuls: bytes per element of A and B (C elements are out_bytes) */
} KINFO[COAST_K_COUNT_] = {
    [COAST_K_CRC16]       = { "crc16",       2,  1,  IN_UNIT_BYTES, 0,  1, 1 },
    [COAST_K_SHA256]      = { "sha256",      32, 32, IN_UNIT_BYTES, 0,  1, 1 },
    [COAST_K_AES128]      = { "aes128",      16, 16, 16,            16, 0, 1 },
    [COAST_K_MM_U32]      = { "mm_u32",      4,  1,  0,             0,  1, 0, 4 },
    [COAST_K_GEMM_TF32]   = { "gemm_tf32",   4,  1,  0,             0,  0, 0, 4 },
    [COAST_K_QSORT]       = { "qsort",       0,  0,  IN_UNIT_BYTES, 0,  0, 0 },
    [COAST_K_CHSTONE_SHA] = { "chstone_sha", 20, 5,  IN_UNIT_BYTES, 0,  0, 1 },
    [COAST_K_CHSTONE_AES] = { "chstone_aes", 64, 16, 64,            64, 0, 1 },
    [COAST_K_GEMM_BF16]   = { "gemm_bf16",   4,  1,  0,             0,  0, 0, 2 },
    [COAST_K_GEMM_FP8]    = { "gemm_fp8",    4,  1,  0,             0,  0, 0, 1 },
    [COAST_K_GEMM_I8]     = { "gemm_i8",     4,  1,  0,             0,  0, 0, 1 },
    [COAST_K_GEMM_F16]    = { "gemm_f16",    4,  1,  0,             0,  0, 0, 2 },
};
/* an id with a row above; the ids between are unassigned (9, 11, 13) and unknown like those past the table */
static int known_kernel(uint32_t kernel) { return kernel < COAST_K_COUNT_ && KINFO[kernel].name; }
static int is_matmul(uint32_t kernel) { return known_kernel(kernel) && KINFO[kernel].mm_elem != 0; }

static int store_votes_wanted(uint32_t fl) {
    return (fl & (COAST_F_STORE_DATA_SYNC | COAST_F_NO_MEM_REPLICATION)) && !(fl & COAST_F_NO_STORE_DATA_SYNC);
}
static int store_votes_built(uint32_t kernel) { return known_kernel(kernel) && KINFO[kernel].store_votes; }

uint32_t coast_flags_honoured(uint32_t kernel, uint32_t nc, uint32_t fl) {
    uint32_t h = fl & (COAST_F_COUNT_ERRORS | COAST_F_COUNT_SYNCS | COAST_F_VERBOSE | COAST_F_MAJORITY_VOTER);
    /* layout: every kernel's native replica placement is the interleaved one (adjacent lanes of a warp; the tensor-core kernels
     * issue the replicas' MMAs back to back per k-step), so -i is what they do; replicas on separate warps (-s) exist for SHA-256 TMR only */
    h |= fl & COAST_F_INTERLEAVE;
    if (kernel == COAST_K_SHA256 && nc == 3) h |= fl & COAST_F_SEGMENT;
    if (store_votes_built(kernel))
        h |= fl & (COAST_F_NO_MEM_REPLICATION | COAST_F_STORE_DATA_SYNC | COAST_F_NO_STORE_DATA_SYNC);
    else if (!store_votes_wanted(fl))
        h |= fl & (COAST_F_NO_STORE_DATA_SYNC);              /* asking for less than what is not there is honoured trivially */
    return h;
}

int coast_set_opt_passes(const char* s) {
    uint32_t nc, fl; int rc = coast_parse_opt_passes(s, &nc, &fl);
    if (rc) return rc;
    G.def_nc = nc; G.def_flags = fl; G.def_set = 1;
    return COAST_OK;
}

/* ------------------------------------------------------------------ */
/* geometry shared with oracle/ by specification (DESIGN.md)            */
/* ------------------------------------------------------------------ */
static uint32_t sha_blocks(uint32_t len) { return (len + 8u) / 64u + 1u; }

uint32_t coast_fault_sites(uint32_t kernel, uint32_t unit_bytes, uint32_t K) {
    switch (kernel) {
    case COAST_K_CRC16:     return 2u * unit_bytes;
    case COAST_K_SHA256:    return 536u * sha_blocks(unit_bytes);
    case COAST_K_AES128:    return 176u;
    case COAST_K_MM_U32:    return K;
    case COAST_K_GEMM_TF32: return 1u;
    case COAST_K_GEMM_BF16: return 1u;
    case COAST_K_GEMM_FP8:  return 1u;
    case COAST_K_GEMM_I8:   return 1u;
    case COAST_K_GEMM_F16:  return 1u;
    case COAST_K_QSORT:     return 33u * (unit_bytes / 4u);
    case COAST_K_CHSTONE_SHA: return 421u * (unit_bytes / 64u + 1u);
    case COAST_K_CHSTONE_AES: return 176u;
    default:                return 0u;
    }
}
uint32_t coast_fault_site_bits(uint32_t kernel, uint32_t unit_bytes, uint32_t K, uint32_t site) {
    (void)K;
    if (kernel == COAST_K_CRC16) return site < unit_bytes ? 16u : 8u;
    if (kernel == COAST_K_AES128 || kernel == COAST_K_CHSTONE_AES) return 8u;
    return 32u;
}
uint32_t coast_out_bytes_per_unit(uint32_t kernel) { return known_kernel(kernel) ? KINFO[kernel].out_bytes : 0; }
uint32_t coast_votes_per_unit(uint32_t kernel) { return known_kernel(kernel) ? KINFO[kernel].votes : 0; }
uint32_t coast_out_bytes(uint32_t kernel, uint32_t unit_bytes) {
    return kernel == COAST_K_QSORT ? unit_bytes : coast_out_bytes_per_unit(kernel);
}
static uint64_t in_bytes_per_unit(const coast_launch_desc* d) {
    if (!known_kernel(d->kernel)) return 0;
    return KINFO[d->kernel].in_bytes == IN_UNIT_BYTES ? d->unit_bytes : KINFO[d->kernel].in_bytes;
}
/* bytes of per-unit aux data the host call stages next to the input (AES keys) */
static uint64_t aux_bytes_per_unit(const coast_launch_desc* d) {
    return known_kernel(d->kernel) && (d->mode & COAST_AES_KEY_PER_UNIT) ? KINFO[d->kernel].key_bytes : 0;
}

/* ------------------------------------------------------------------ */
/* the launch                                                           */
/* ------------------------------------------------------------------ */
/* A tensor map is a pure function of its description.  The host-call path re-creates the same handful of row maps every call,
 * so `cached` maps are looked up among the last 16 (round-robin replacement). */
static int encode_map(const map_desc* want, CUdeviceptr scratch, int cached, CUtensorMap* map) {
    map_desc m = *want;
    if (m.in_scratch) { m.base += scratch; m.in_scratch = 0; }
    if (cached)
        for (int i = 0; i < G.n_tmaps; ++i)
            if (!memcmp(&G.tmaps[i].key, &m, sizeof m)) { *map = G.tmaps[i].map; return COAST_OK; }
    static const cuuint32_t estr[3] = { 1, 1, 1 };
    DRV(p_cuTensorMapEncodeTiled(map, m.dtype, m.rank, (void*)m.base, m.dim, m.stride, m.box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 m.swz, m.l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
    if (cached) {
        const int n_slots = (int)(sizeof G.tmaps / sizeof G.tmaps[0]);
        int k = G.n_tmaps < n_slots ? G.n_tmaps++ : (G.tmap_next++ % n_slots);
        G.tmaps[k].key = m; G.tmaps[k].map = *map;
    }
    return COAST_OK;
}

/* One row per matmul operand type: what the GEMM launch and the kernel names need to know about it (MM_U32: its names only). */
static const struct mm_op {
    const char* ty;                         /* the type in messages: GEMM_<ty> */
    const char* prefix, * stem;             /* kernel names: xmr_<prefix>_<stem>...; scaled and 16-bit-output GEMMs swap the prefix */
    unsigned bk;                            /* elements per k-block (one 128-byte swizzle row) */
    CUtensorMapDataType dt;                 /* A's and B's tensor-map element type */
    int b_in_place;                         /* B (K x N) is read in place, MN-major: no transposing pre-pass, no scratch */
    int bt_kernels;                         /* a caller's B^T has kernels of its own (_bt); else the same kernels read it */
    int nc_first;                           /* _nc<n>_inj<i> on the kernels that are neither grouped nor _bt (they came first) */
    int grp_variant;                        /* grouped kernels keep the path variant (the n of NC 1); else they carry none */
    const char* c16;                        /* the prefix of the kernels with a 2-byte C: o16 (bfloat16), h16 (f16); NULL: none */
} MM_OPS[COAST_K_COUNT_] = {
    [COAST_K_MM_U32]    = { "U32",  "mm",   "u32",  0,                0,                                0, 1, 1, 1 },
    [COAST_K_GEMM_TF32] = { "TF32", "gemm", "tf32", XMR_GEMM_BK,      CU_TENSOR_MAP_DATA_TYPE_FLOAT32,  0, 0, 1, 1 },
    [COAST_K_GEMM_BF16] = { "BF16", "gemm", "bf16", XMR_GEMM_BF16_BK, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 1, 1, 0, 1, "o16" },
    [COAST_K_GEMM_FP8]  = { "FP8",  "gemm", "fp8",  XMR_GEMM_FP8_BK,  CU_TENSOR_MAP_DATA_TYPE_UINT8,    0, 0, 0, 0, "o16" },
    [COAST_K_GEMM_I8]   = { "I8",   "gemm", "i8",   XMR_GEMM_FP8_BK,  CU_TENSOR_MAP_DATA_TYPE_UINT8,    0, 0, 0, 0 },
    /* written with designators: GEMM_BF16's layout with IEEE binary16 elements.  (tests/test_abi.py pins the positional rows
     * above; tests/test_gemm_f16_host_logic.py checks this one.) */
    [COAST_K_GEMM_F16]  = { .ty = "F16", .prefix = "gemm", .stem = "f16", .bk = XMR_GEMM_BF16_BK, .dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                            .b_in_place = 1, .bt_kernels = 1, .nc_first = 0, .grp_variant = 1, .c16 = "h16" },
};

/* The shape of a matmul launch, read off its descriptor once.  Batched (COAST_MM_BATCHED): the stacked A and C are one
 * (batch*M)-row matrix and only B changes from one product to the next.  Grouped (COAST_MM_GROUPED): M is the product count G,
 * the stacked A and C are one R-row matrix from row ro[0] (R = n_units / N) and B is G matrices end to end. */
typedef struct {
    unsigned es;                  /* bytes per element of A and B */
    unsigned ces;                 /* bytes per element of C: 4, or 2 with COAST_MM_OUT_BF16 (bfloat16) or COAST_MM_OUT_F16 (f16) */
    int batched, grouped, bt;     /* the mode bits */
    uint64_t P;                   /* products: 1, the batch or G */
    uint64_t rows;                /* stacked rows of A and C: batch*M or R */
    int b_rows_k;                 /* B's map has K rows per product (GEMM_BF16 reading B in place); every B^T map has N (GEMM_FP8's
                                     and GEMM_I8's always: a B^T map over the pre-pass's scratch or the caller's B^T) */
    uint32_t b_rows;              /* rows per product of B's map */
    int scaled, rowwise;          /* GEMM_FP8 with COAST_MM_SCALE_TENSOR or COAST_MM_SCALE_ROWWISE; the latter */
} mm_shape;

/* What kernel selection decides about a launch; run_plan() does the rest. */
typedef struct launch_plan launch_plan;
struct launch_plan {
    char name[64];
    unsigned block, smem;
    uint64_t ctas;                /* CTAs the work needs (0: one warp per 32/nc units, the lane-interleaved kernels) */
    unsigned waves;               /* the grid is at most this many waves of resident CTAs; 0: all ctas */
    unsigned cluster;             /* CTAs per cluster: the grid is a multiple of it */
    int n_maps, cache_maps;       /* tensor maps: kernel parameters 2 and 3 */
    map_desc map[2];
    size_t scratch;               /* stream-ordered scratch for the pre-pass and the maps */
    size_t scratch_per_cta;       /* plus this much per CTA of the grid, handed to the kernel as xmr_args.aux */
    int scratch_as_aux;           /* hand the scratch to the kernel as xmr_args.aux even without per-CTA scratch */
    int (*prepass)(const launch_plan* L, const coast_launch_desc* d, CUdeviceptr scratch, CUstream s);
    mm_shape mm;                  /* the matmuls */
    /* grouped matmuls: the kernel takes the row offsets and the group block (at grp_off in scratch) after its maps; the scan
     * pre-pass cuts the products into tiles of grp_tm rows, grp_tiles_n per tile row (grp_tm 0: no scan, the plain kernel) */
    size_t grp_off;
    unsigned grp_tm, grp_tiles_n;
};

/* The TMA-ring kernels: tiles of tile_rows units of row_bytes each, loaded as equal boxes of at most 256 rows.  With a row
 * pack shift p the same dense bytes are described as rows 2^p times longer. */
static void plan_ring(launch_plan* L, xmr_args* a, unsigned tile_rows, unsigned row_bytes, unsigned pack, CUtensorMapSwizzle swz) {
    L->ctas = (a->n_units + tile_rows - 1) / tile_rows;
    L->waves = 1;
    a->n_tiles = (unsigned)L->ctas;
    L->n_maps = 1; L->cache_maps = 1;
    map_desc* m = &L->map[0];
    m->dtype = CU_TENSOR_MAP_DATA_TYPE_UINT32; m->rank = 2; m->base = (uintptr_t)a->in;
    m->dim[0] = m->box[0] = (row_bytes << pack) / 4u;
    m->dim[1] = a->n_units >> pack;
    m->stride[0] = row_bytes << pack;
    m->box[1] = (tile_rows / xmr_ring_loads(tile_rows)) >> pack;
    m->swz = swz; m->l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
}

/* A K-major operand of the wgmma kernels, 128-byte swizzle: rows x K elements of esize bytes, in `planes` planes (or any dense
 * row-major matrix of `rows` rows of K elements, loaded in boxes of 128 bytes x box_rows: GEMM_BF16's B). */
static void plan_wg_map(map_desc* m, CUtensorMapDataType dtype, unsigned esize, uintptr_t base, int in_scratch, uint32_t K,
                        uint32_t rows, unsigned planes, unsigned box_rows) {
    m->dtype = dtype; m->rank = planes > 1 ? 3 : 2; m->base = base; m->in_scratch = in_scratch;
    m->dim[0] = K; m->dim[1] = rows; m->dim[2] = planes;
    m->stride[0] = (cuuint64_t)K * esize; m->stride[1] = (cuuint64_t)rows * K * esize;
    m->box[0] = 128u / esize; m->box[1] = box_rows; m->box[2] = planes;
    m->swz = CU_TENSOR_MAP_SWIZZLE_128B; m->l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
}

/* rows of the stacked operands are tensor-map coordinates: A's rows and B's P * b_rows */
static int mm_rows_fit(const mm_shape* m) { return m->rows < (1ull << 31) && m->P * m->b_rows < (1ull << 31); }

/* a matmul mode bit on another kernel */
static int mm_bit_refused(const coast_launch_desc* d, uint32_t bit) {
    if (!(d->mode & bit) || is_matmul(d->kernel)) return COAST_OK;
    const char* what = bit == COAST_MM_BATCHED ? "COAST_MM_BATCHED: batched products exist"
                     : bit == COAST_MM_GROUPED ? "COAST_MM_GROUPED: grouped products exist" : "COAST_MM_B_TRANSPOSED: a transposed B exists";
    return fail(COAST_ERR_BAD_ARG, "%s for MM_U32, GEMM_TF32 and GEMM_BF16 only, plus GEMM_FP8 and GEMM_I8 (kernel %u)", what, d->kernel);
}
/* The scale bits (GEMM_FP8 only): one of the two, both scale pointers, d_scale_a 4-byte aligned and, row-wise, d_scale_b
 * 8-byte aligned (the kernels read a thread's two column scales as one float2) */
static int mm_scale_check(const coast_launch_desc* d) {
    const uint32_t bits = d->mode & (COAST_MM_SCALE_TENSOR | COAST_MM_SCALE_ROWWISE);
    if (!bits) return COAST_OK;
    const char* what = bits == COAST_MM_SCALE_TENSOR ? "COAST_MM_SCALE_TENSOR" : "COAST_MM_SCALE_ROWWISE";
    if (d->kernel != COAST_K_GEMM_FP8)
        return fail(COAST_ERR_BAD_ARG, "%s: scaled products exist for GEMM_FP8 only (kernel %u)",
                    bits == (COAST_MM_SCALE_TENSOR | COAST_MM_SCALE_ROWWISE) ? "COAST_MM_SCALE_TENSOR / COAST_MM_SCALE_ROWWISE" : what, d->kernel);
    if (bits == (COAST_MM_SCALE_TENSOR | COAST_MM_SCALE_ROWWISE))
        return fail(COAST_ERR_BAD_ARG, "COAST_MM_SCALE_TENSOR and COAST_MM_SCALE_ROWWISE cannot be combined: one scale layout per launch");
    if (!d->d_scale_a || !d->d_scale_b)
        return fail(COAST_ERR_BAD_ARG, "%s: d_scale_a and d_scale_b must point to the scales of A and B", what);
    if (((uintptr_t)d->d_scale_a) & 3u) return fail(COAST_ERR_BAD_ARG, "%s: d_scale_a must be 4-byte aligned", what);
    if (bits == COAST_MM_SCALE_ROWWISE && (((uintptr_t)d->d_scale_b) & 7u))
        return fail(COAST_ERR_BAD_ARG, "COAST_MM_SCALE_ROWWISE: d_scale_b must be 8-byte aligned (column scales are read in pairs)");
    return COAST_OK;
}
/* BF16 output (GEMM_BF16 and GEMM_FP8 only; not with a scale bit) and FP16 output (GEMM_F16 only; not with BF16 output) */
static int mm_out_check(const coast_launch_desc* d) {
    if (d->mode & COAST_MM_OUT_F16) {
        if (d->kernel != COAST_K_GEMM_F16)
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_OUT_F16: float16 output exists for GEMM_F16 only (kernel %u)", d->kernel);
        if (d->mode & COAST_MM_OUT_BF16)
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_OUT_F16 and COAST_MM_OUT_BF16 cannot be combined: one C type per launch");
    }
    if (!(d->mode & COAST_MM_OUT_BF16)) return COAST_OK;
    if (d->kernel != COAST_K_GEMM_BF16 && d->kernel != COAST_K_GEMM_FP8)
        return fail(COAST_ERR_BAD_ARG, "COAST_MM_OUT_BF16: bfloat16 output exists for GEMM_BF16 and GEMM_FP8 only (kernel %u)", d->kernel);
    if (d->mode & (COAST_MM_SCALE_TENSOR | COAST_MM_SCALE_ROWWISE))
        return fail(COAST_ERR_UNSUPPORTED, "COAST_MM_OUT_BF16: scaled GEMM_FP8 has no bfloat16-output kernels yet; its C is fp32");
    return COAST_OK;
}
/* The checks shared by coast_launch and coast_run_host: a matmul mode bit on another kernel, the scale and output bits, then the
 * shape of a batch or of groups.  Fills *m for the matmul kernels; m->ces is the one place that knows C's element size. */
static int mm_check(const coast_launch_desc* d, mm_shape* m) {
    int rc;
    memset(m, 0, sizeof *m);
    if ((rc = mm_bit_refused(d, COAST_MM_BATCHED)) || (rc = mm_bit_refused(d, COAST_MM_GROUPED)) ||
        (rc = mm_bit_refused(d, COAST_MM_B_TRANSPOSED)) || (rc = mm_scale_check(d)) || (rc = mm_out_check(d)))
        return rc;
    if (!is_matmul(d->kernel)) return COAST_OK;
    m->ces = (d->mode & (COAST_MM_OUT_BF16 | COAST_MM_OUT_F16)) ? 2u : KINFO[d->kernel].out_bytes;
    m->scaled = (d->mode & (COAST_MM_SCALE_TENSOR | COAST_MM_SCALE_ROWWISE)) != 0;
    m->rowwise = (d->mode & COAST_MM_SCALE_ROWWISE) != 0;
    m->es = KINFO[d->kernel].mm_elem;
    m->batched = (d->mode & COAST_MM_BATCHED) != 0;
    m->grouped = (d->mode & COAST_MM_GROUPED) != 0;
    m->bt = (d->mode & COAST_MM_B_TRANSPOSED) != 0;
    m->b_rows_k = MM_OPS[d->kernel].b_in_place && !m->bt;
    m->b_rows = m->b_rows_k ? d->K : d->N;
    const char bc = m->b_rows_k ? 'K' : 'N';
    m->P = 1; m->rows = d->M;
    if (m->batched) {
        if (!d->M || !d->N || !d->K) return fail(COAST_ERR_BAD_ARG, "COAST_MM_BATCHED: M, N and K are the shape of one product and must be nonzero");
        const uint64_t mn = (uint64_t)d->M * d->N;
        if (!d->n_units || d->n_units % mn)
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_BATCHED: n_units must be a nonzero multiple of M*N = %llu (got %llu)",
                        (unsigned long long)mn, (unsigned long long)d->n_units);
        m->P = d->n_units / mn; m->rows = m->P * d->M;
        if (!mm_rows_fit(m))
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_BATCHED: batch*M and batch*%c must be below 2^31 (batch %llu, M %u, %c %u)",
                        bc, (unsigned long long)m->P, d->M, bc, m->b_rows);
    }
    if (m->grouped) {
        if (d->mode & (COAST_MM_BATCHED | COAST_UNIT_OFFSETS))
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: cannot be combined with COAST_MM_BATCHED or COAST_UNIT_OFFSETS");
        if (!d->M || d->M > XMR_MM_GRP_MAX)
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: M is the product count G, 1..%u (got %u)", XMR_MM_GRP_MAX, d->M);
        if (!d->N || !d->K) return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: N and K are shared by every product and must be nonzero");
        if (d->n_units % d->N)
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: n_units must be a multiple of N = %u (R rows x N; got %llu)", d->N,
                        (unsigned long long)d->n_units);
        m->P = d->M; m->rows = d->n_units / d->N;
        if (!mm_rows_fit(m))
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: the rows R and G*%c must be below 2^31 (R %llu, G %u, %c %u)",
                        bc, (unsigned long long)m->rows, d->M, bc, m->b_rows);
        if (!d->d_rows || (((uintptr_t)d->d_rows) & 7u))
            return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: d_rows must point to G + 1 8-byte aligned uint64_t row offsets");
    }
    return COAST_OK;
}
/* tiles of bm rows over the stacked rows; a grouped launch's products start anywhere, so it gets one more per product (a bound) */
static uint64_t mm_row_tiles(const mm_shape* m, unsigned bm) { return m->rows / bm + (m->grouped ? m->P : 0); }

/* A matmul kernel's name: xmr_<prefix>_<stem><variant>[_bt][_grp], then _inj<i>_nc<n>, or _nc<n>_inj<i> where the row says so.
 * The prefix is scaled for COAST_MM_SCALE_* and the row's c16 for a 2-byte C (o16: COAST_MM_OUT_BF16, h16: COAST_MM_OUT_F16); the
 * variant is the path ("n", "p", "_tc", "_tiled" or ""). */
static void mm_kernel_name(char* name, uint32_t kernel, const char* variant, int bt, int grouped, int scaled, int c16, uint32_t nc, int inj) {
    const struct mm_op* op = &MM_OPS[kernel];
    bt = bt && op->bt_kernels;
    const int ni = op->nc_first && !bt && !grouped;
    snprintf(name, 64, "xmr_%s_%s%s%s%s_%s%u_%s%u", scaled ? "scaled" : c16 ? op->c16 : op->prefix, op->stem,
             grouped && !op->grp_variant ? "" : variant, bt ? "_bt" : "", grouped ? "_grp" : "", ni ? "nc" : "inj", ni ? nc : (unsigned)inj,
             ni ? "inj" : "nc", ni ? (unsigned)inj : nc);
}

/* Pre-passes of the wgmma kernels: TF32, FP8 and INT8 wgmma read both operands K-major, so B (K x N, row-major) is transposed into
 * scratch (4-byte or 1-byte elements);
 * the limb kernel splits A and B into u8 limb planes ([plane][rows][K] and, transposed, [plane][P N][K]).  The products' B
 * matrices become one stacked (P N) x K operand; their A matrices already are one matrix. */
static int prepass_transpose_b(const launch_plan* L, const coast_launch_desc* d, CUdeviceptr bt, CUstream s) {
    const void* B = d->d_aux; unsigned int k32 = d->K, n32 = d->N, nb = (unsigned)L->mm.P;
    void* params[] = { &B, &bt, &k32, &n32, &nb };
    return launch_small(L->mm.es == 1 ? "xmr_gemm_bt_u8" : "xmr_gemm_bt", (unsigned)G.sm_count * 8u, XMR_PREPASS_THREADS, params, s);
}
/* A's rows (groups: the R rows from row ro[0]), then the B^T planes [plane][p N + n][k]: split_bt transposes B; a caller's B^T
 * (COAST_MM_B_TRANSPOSED) already has that row order, so the streaming split of A makes them from its (P N) rows of K. */
static int prepass_split_limbs(const launch_plan* L, const coast_launch_desc* d, CUdeviceptr pa, CUstream s) {
    unsigned long long rows = L->mm.rows, K = d->K; const void* A = d->d_in; const void* ro = d->d_rows; const void* B = d->d_aux;
    void* params_a[] = { &A, &pa, &rows, &K };
    void* params_grp[] = { &ro, &A, &pa, &rows, &K };
    int rc = launch_small(L->mm.grouped ? "xmr_mm_grp_split_a" : "xmr_mm_split_a", (unsigned)G.sm_count * 8u, XMR_PREPASS_THREADS,
                          L->mm.grouped ? params_grp : params_a, s);
    if (rc) return rc;
    CUdeviceptr pb = pa + (size_t)rows * d->K * 4u;
    if (L->mm.bt) {
        unsigned long long b_rows = L->mm.P * d->N;
        void* params[] = { &B, &pb, &b_rows, &K };
        return launch_small("xmr_mm_split_a", (unsigned)G.sm_count * 8u, XMR_PREPASS_THREADS, params, s);
    }
    unsigned int k32 = d->K, n32 = d->N, nb = (unsigned)L->mm.P;
    void* params_b[] = { &B, &pb, &k32, &n32, &nb };
    return launch_small("xmr_mm_split_bt", (unsigned)G.sm_count * 8u, XMR_PREPASS_THREADS, params_b, s);
}
/* tile_start of the products (xmr_mm_group_scan, one CTA) into the group block; for TF32, BF16 and FP8 (a_map) it also rebases the host's A map
 * onto row ro[0] of d_in with R rows, so no host-side read of the device table is needed */
static int prepass_group_scan(const launch_plan* L, const coast_launch_desc* d, CUdeviceptr grp, const CUtensorMap* a_map, CUstream s) {
    const void* ro = d->d_rows; const void* base = d->d_in;
    unsigned int n_grp = d->M, R = (unsigned)L->mm.rows, tm = L->grp_tm, tn = L->grp_tiles_n;
    unsigned int row_bytes = a_map ? d->K * L->mm.es : 0u;
    CUtensorMap none; memset(&none, 0, sizeof none);
    void* params[] = { &ro, &n_grp, &R, &tm, &tn, &grp, &base, &row_bytes, (void*)(a_map ? a_map : &none) };
    return launch_small("xmr_mm_group_scan", 1, XMR_MM_GRP_SCAN_THREADS, params, s);
}

/* Ragged batches (COAST_UNIT_OFFSETS): the bound on every length, and the checks shared by coast_launch and coast_run_host. */
static uint32_t ragged_bound_max(uint32_t kernel) {
    return kernel == COAST_K_CRC16 ? 255u : kernel == COAST_K_QSORT ? 4096u : (1u << 28);
}
static int ragged_check(const coast_launch_desc* d) {
    if (d->kernel != COAST_K_SHA256 && d->kernel != COAST_K_CRC16 && d->kernel != COAST_K_QSORT)
        return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: ragged batches exist for CRC16, SHA256 and QSORT only (kernel %u)", d->kernel);
    if (d->unit_bytes > ragged_bound_max(d->kernel))
        return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: unit_bytes bounds every length and is at most %u for %s (got %u)",
                    ragged_bound_max(d->kernel), KINFO[d->kernel].name, d->unit_bytes);
    if (d->kernel == COAST_K_QSORT) {                        /* int32 arrays: whole elements, aligned buffers */
        if (d->unit_bytes == 0 || (d->unit_bytes & 3u))
            return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: quicksort's unit_bytes bounds every array and is a multiple of 4 in "
                                           "4..4096 (got %u)", d->unit_bytes);
        if ((((uintptr_t)d->d_in) & 3u) || (((uintptr_t)d->d_out) & 3u))
            return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: quicksort's d_in and d_out must be 4-byte aligned");
    }
    if (d->n_units >= (1ull << 32)) return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: n_units must be below 2^32");
    if (!d->d_aux || (((uintptr_t)d->d_aux) & 7u))
        return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: d_aux must point to n_units + 1 8-byte aligned uint64_t offsets");
    return COAST_OK;
}

/* Cost-ordering pre-pass of the ragged kernels (xmr_ragged.cuh): zero the header and the bucket counts, histogram, one-CTA scan
 * (which also stores the offset table's address in the header), scatter into the permutation.  All on the launch's stream. */
static int prepass_ragged(const launch_plan* L, const coast_launch_desc* d, CUdeviceptr scratch, CUstream s) {
    (void)L;
    DRV(p_cuMemsetD8Async(scratch, 0, XMR_RAGGED_PERM, s));
    const void* off = d->d_aux;
    unsigned long long n = d->n_units;
    unsigned int bound = d->unit_bytes;
    unsigned int kind = d->kernel == COAST_K_SHA256 ? XMR_RAGGED_COST_SHA : d->kernel == COAST_K_QSORT ? XMR_RAGGED_COST_QSORT
                                                                                                       : XMR_RAGGED_COST_CRC;
    const uint64_t ctas = (n + XMR_CTA_THREADS - 1) / XMR_CTA_THREADS, cap = (uint64_t)G.sm_count * 8u;
    const unsigned grid = (unsigned)(ctas < cap ? ctas : cap);
    void* params[] = { &off, &n, &bound, &kind, &scratch };
    int rc = launch_small("xmr_ragged_hist", grid, XMR_CTA_THREADS, params, s); if (rc) return rc;
    void* params_scan[] = { &off, &scratch };
    rc = launch_small("xmr_ragged_scan", 1, XMR_RAGGED_SCAN_THREADS, params_scan, s); if (rc) return rc;
    return launch_small("xmr_ragged_scatter", grid, XMR_CTA_THREADS, params, s);
}

/* Scratch comes from the stream-ordered pool: allocated on the launch's stream and released on it after the kernel, so launches
 * on different streams never share it, and the pool keeps released memory cached (no driver allocation in steady state). */
static int run_plan(const launch_plan* L, const coast_launch_desc* d, xmr_args* a, CUstream stream) {
    CUfunction fn; int occ = 1;
    int rc = get_fn(L->name, L->smem, L->block, &fn, &occ); if (rc) return rc;
    const uint64_t cap = (uint64_t)G.sm_count * (unsigned)occ * L->waves;
    unsigned grid = (unsigned)(L->waves && L->ctas > cap ? cap : L->ctas);
    grid -= grid % L->cluster;
    const size_t bytes = L->scratch + (size_t)grid * L->scratch_per_cta;
    CUdeviceptr scratch = 0;
    if (bytes) DRV(p_cuMemAllocFromPoolAsync(&scratch, bytes, G.pool, stream));
    if (L->scratch_per_cta || L->scratch_as_aux) a->aux = (const void*)scratch;
    CUtensorMap maps[2];
    rc = L->prepass ? L->prepass(L, d, scratch, stream) : COAST_OK;
    for (int i = 0; i < L->n_maps && !rc; ++i) rc = encode_map(&L->map[i], scratch, L->cache_maps, &maps[i]);
    /* grouped: the tile table (and the GEMMs' rebased A map) after the other pre-passes; the kernel takes ro and the group block,
     * then a scaled kernel the scales */
    const void* ro = d->d_rows; const void* sa = d->d_scale_a; const void* sb = d->d_scale_b;
    CUdeviceptr grp = scratch + L->grp_off;
    if (!rc && L->mm.grouped && L->grp_tm)
        rc = prepass_group_scan(L, d, grp, d->kernel != COAST_K_MM_U32 ? &maps[0] : NULL, stream);
    if (!rc) {
        void* params[7] = { a };
        int n_params = 1;
        for (int i = 0; i < L->n_maps; ++i) params[n_params++] = &maps[i];
        if (L->mm.grouped) { params[n_params++] = &ro; params[n_params++] = &grp; }
        if (L->mm.scaled) { params[n_params++] = &sa; params[n_params++] = &sb; }
        if (d->flags & COAST_F_VERBOSE)
            fprintf(stderr, "coast_rt: %s grid=%u block=%u smem=%u units=%llu\n", L->name, grid, L->block, L->smem,
                    (unsigned long long)d->n_units);
        CUresult r = p_cuLaunchKernel(fn, grid, 1, 1, L->block, 1, 1, L->smem, stream, params, NULL);
        if (r != CUDA_SUCCESS) rc = drv_fail(r, "cuLaunchKernel");
    }
    if (scratch) p_cuMemFreeAsync(scratch, stream);
    return rc;
}

static int launch_impl(const coast_launch_desc* d, void* stream) {
    int rc = ensure_ctx(); if (rc) return rc;
    if (!d) return fail(COAST_ERR_BAD_ARG, "null descriptor");
    if (!known_kernel(d->kernel)) return fail(COAST_ERR_BAD_ARG, "unknown kernel id %u", d->kernel);
    if (d->num_clones < 1 || d->num_clones > 3) return fail(COAST_ERR_BAD_ARG, "num_clones must be 1, 2 (DWC) or 3 (TMR)");
    const int ragged = (d->mode & COAST_UNIT_OFFSETS) != 0;
    if (ragged && (rc = ragged_check(d))) return rc;
    mm_shape m;
    if ((rc = mm_check(d, &m))) return rc;
    if (d->n_units == 0) return COAST_OK;
    if (!d->d_in || !d->d_out) return fail(COAST_ERR_BAD_ARG, "null device buffer");
    const uint32_t nc = d->num_clones;
    const uint32_t upw = xmr_units_per_warp(nc);
    const int inj = d->plan && d->plan->mode != COAST_PLAN_NONE;

    xmr_args a; memset(&a, 0, sizeof a);
    a.in = d->d_in; a.out = d->d_out; a.aux = d->d_aux;
    a.n_units = d->n_units; a.unit_base = d->unit_base;
    a.counters = (unsigned long long*)(G.peer_counters ? G.peer_counters : G.counters);
    a.status = (unsigned char*)d->d_status;
    /* the kernels find a batch from n_units / N (rows of the stacked problem) and a.M (rows per product): a batch of one is
     * an unbatched launch, argument block included */
    a.unit_bytes = d->unit_bytes; a.flags = d->flags; a.mode = d->mode & ~(COAST_MM_BATCHED | COAST_MM_GROUPED | COAST_MM_B_TRANSPOSED |
                                                                      COAST_MM_SCALE_TENSOR | COAST_MM_SCALE_ROWWISE | COAST_MM_OUT_BF16 |
                                                                      COAST_MM_OUT_F16);
    if (m.rowwise) a.mode |= XMR_MODE_SCALE_ROWWISE;
    a.M = d->M; a.N = d->N; a.K = d->K;
    memcpy(a.key, d->key, 16);
    if (inj) {
        a.plan_mode = d->plan->mode; a.seed_lo = d->plan->seed_lo; a.seed_hi = d->plan->seed_hi;
        a.threshold = d->plan->threshold; a.plan_table = (const unsigned int*)d->plan->d_table;
        if (a.plan_mode == COAST_PLAN_TABLE && !a.plan_table) return fail(COAST_ERR_BAD_ARG, "TABLE plan without d_table");
        if (a.plan_mode > COAST_PLAN_TABLE) return fail(COAST_ERR_BAD_ARG, "unknown fault plan mode %u", a.plan_mode);
    }
    a.n_sites = coast_fault_sites(d->kernel, d->unit_bytes, d->K);
    /* in-loop store votes (-storeDataSync / -noMemReplication): built for CRC16, SHA256 and MM_U32, loud everywhere else */
    const int store_votes = store_votes_wanted(d->flags) && nc > 1;
    if (store_votes && !store_votes_built(d->kernel)) {
        const char* strict = getenv("COAST_STRICT_FLAGS");
        if (strict && strcmp(strict, "0"))
            return fail(COAST_ERR_UNSUPPORTED, "-noMemReplication / -storeDataSync: the %s kernel has no in-loop store votes "
                                               "(COAST_STRICT_FLAGS is set)", KINFO[d->kernel].name);
        if (!(G.warned_store_votes & (1u << d->kernel))) {
            G.warned_store_votes |= 1u << d->kernel;
            fprintf(stderr, "coast_rt: WARNING: -noMemReplication / -storeDataSync are NOT honoured by the %s kernel: it has no in-loop "
                            "store votes and runs the default sync set (SoR-exit votes only).  COAST_STRICT_FLAGS=1 makes this an error.\n",
                    KINFO[d->kernel].name);
        }
    }
    if (store_votes && store_votes_built(d->kernel)) a.flags |= XMR_F_STORE_VOTES;

    /* kernel selection: name, CTA, shared memory, grid rule, tensor maps, pre-pass and scratch (xmr_geom.h) */
    launch_plan L; memset(&L, 0, sizeof L);
    L.block = XMR_CTA_THREADS; L.waves = 4; L.cluster = 1;
    const int aligned16 = (((uintptr_t)d->d_in) & 15u) == 0;
    const int ring_ok = d->unit_bytes == 64 && aligned16 && d->n_units < 0x7FFFFF00ull && !store_votes;   /* 64-byte rows through TMA */
    L.mm = m;
    if (is_matmul(d->kernel)) {
        const char* fam = d->kernel == COAST_K_MM_U32 ? "MM" : "GEMM";
        if (!d->d_aux || !d->M || !d->N || !d->K) return fail(COAST_ERR_BAD_ARG, "%s needs A (d_in), B (d_aux) and M,N,K", fam);
        if (!m.batched && !m.grouped && d->n_units != (uint64_t)d->M * d->N) return fail(COAST_ERR_BAD_ARG, "%s: n_units must be M*N", fam);
    }
    switch (d->kernel) {
    case COAST_K_SHA256:
        if (((uintptr_t)d->d_out) & 15u) return fail(COAST_ERR_BAD_ARG, "SHA output must be 16-byte aligned");
        if (ragged) {
            snprintf(L.name, sizeof L.name, "xmr_sha256_var_inj%d_nc%u", inj, nc);
        } else if (!ring_ok) {
            snprintf(L.name, sizeof L.name, "xmr_sha256_gen_nc%u_inj%d", nc, inj);
        } else if (nc == 3 && !(d->flags & COAST_F_INTERLEAVE)) {
            /* TMR replica scheduling: -s (segmented, the reference default, interface.cpp:245-247) = replicas on
             * adjacent warps; -i (interleaved) = replicas on adjacent lanes.  Results are identical. */
            snprintf(L.name, sizeof L.name, "xmr_sha256_b64_seg_nc3_inj%d", inj);
            L.block = XMR_SHA_SEG_THREADS; L.smem = xmr_sha_seg_smem();
            plan_ring(&L, &a, XMR_SHA_SEG_TILE_ROWS, 64, 0, CU_TENSOR_MAP_SWIZZLE_64B);
        } else {
            snprintf(L.name, sizeof L.name, "xmr_sha256_b64_nc%u_inj%d", nc, inj);
            L.smem = xmr_sha_smem(nc);
            plan_ring(&L, &a, xmr_sha_tile_rows(nc), 64, 0, CU_TENSOR_MAP_SWIZZLE_64B);
        }
        break;
    case COAST_K_CRC16:
        if (ragged) {
            snprintf(L.name, sizeof L.name, "xmr_crc16_var_inj%d_nc%u", inj, nc);
            break;
        }
        if (d->unit_bytes < 1 || d->unit_bytes > 255) return fail(COAST_ERR_BAD_ARG, "crc16 length is an unsigned char (1..255)");
        if (ring_ok) {                                      /* table kernel: byte-step table and tile ring in shared memory */
            snprintf(L.name, sizeof L.name, "xmr_crc16_b64_nc%u_inj%d", nc, inj);
            L.block = xmr_crc_threads(nc); L.smem = xmr_crc_smem(nc);
            plan_ring(&L, &a, xmr_crc_tile_rows(nc), 64, 0, CU_TENSOR_MAP_SWIZZLE_64B);
        } else {
            snprintf(L.name, sizeof L.name, "xmr_crc16_gen_nc%u_inj%d", nc, inj);
        }
        break;
    case COAST_K_AES128: {
        const int dec = (d->mode & COAST_AES_DECRYPT) != 0, perkey = (d->mode & COAST_AES_KEY_PER_UNIT) != 0;
        if (perkey && !d->d_aux) return fail(COAST_ERR_BAD_ARG, "per-unit keys need d_aux");
        if (!aligned16 || (((uintptr_t)d->d_out) & 15u)) return fail(COAST_ERR_BAD_ARG, "AES buffers must be 16-byte aligned");
        if (perkey && (((uintptr_t)d->d_aux) & 15u)) return fail(COAST_ERR_BAD_ARG, "AES per-unit keys must be 16-byte aligned");
        if (d->n_units >= 0x7FFFFF00ull) return fail(COAST_ERR_UNSUPPORTED, "AES: at most 2^31 - 257 blocks per launch (split the batch)");
        /* one table-driven body (xmr_aes128.cuh): enc / dec with one ECB key, enck / deck with per-unit keys */
        static const char* const stem[4] = { "xmr_aes128_enc", "xmr_aes128_dec", "xmr_aes128_enck", "xmr_aes128_deck" };
        snprintf(L.name, sizeof L.name, "%s_nc%u_inj%d", stem[dec + 2 * perkey], nc, inj);
        L.block = XMR_AES_THREADS; L.smem = xmr_aes_smem(dec);
        /* the same dense bytes as 256- or 64-byte rows when the count allows */
        const unsigned tile_rows = xmr_aes_tile_rows(nc), box_rows = tile_rows / xmr_ring_loads(tile_rows);
        unsigned pack = d->n_units % 16u == 0 ? 4u : d->n_units % 4u == 0 ? 2u : 0u;
        while (pack && box_rows % (1u << pack)) pack -= 2u;
        a.mode = (a.mode & ~(XMR_MODE_AES_ROWPACK_MASK << XMR_MODE_AES_ROWPACK_SHIFT)) | (pack << XMR_MODE_AES_ROWPACK_SHIFT);
        plan_ring(&L, &a, tile_rows, 16, pack, CU_TENSOR_MAP_SWIZZLE_NONE);
        break;
    }
    case COAST_K_MM_U32: {
        /* the plain kernel (one lane per replica per element) takes any shape and the per-k votes on `sum`; tile-aligned problems
         * go to the tensor cores (exact, u8 limbs on wgmma) or the register-tiled kernel; COAST_MM_PATH=tc|tiled|naive overrides.
         * The shape rules are those of one product; a batch stacks the products' rows (no tile straddles two of them), and the
         * rows of grouped products are free. */
        const char* path = getenv("COAST_MM_PATH");
        const int aligned = aligned16 && !(((uintptr_t)d->d_aux) & 15u) && !(((uintptr_t)d->d_out) & 15u);
        const int tiles_ok = !store_votes && aligned;
        const char* variant = "";
        int bt_name = m.bt;
        if (tiles_ok && (!path || !strcmp(path, "tc")) && (m.grouped || d->M % XMR_WG_BM == 0) && d->N % xmr_mmtc_bn(1) == 0 &&
            d->K % XMR_MMTC_BK == 0) {
            const unsigned bn = xmr_mmtc_bn(nc);
            variant = "_tc";
            bt_name = m.bt && inj;                           /* B^T: the same planes (the pre-pass differs); only the fault recompute reads B itself */
            L.block = XMR_WG_THREADS; L.smem = xmr_mmtc_smem(nc);
            L.ctas = mm_row_tiles(&m, XMR_WG_BM) * (d->N / bn); L.waves = 1;           /* persistent CTAs */
            L.scratch = ((size_t)m.rows * d->K + (size_t)m.P * d->K * d->N) * 4u;       /* 4 planes of 1 byte per element */
            L.prepass = prepass_split_limbs;
            L.grp_tm = XMR_WG_BM; L.grp_tiles_n = d->N / bn;
            L.n_maps = 2;
            plan_wg_map(&L.map[0], CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, 0, 1, d->K, (uint32_t)m.rows, 4, XMR_WG_BM);
            plan_wg_map(&L.map[1], CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, (size_t)m.rows * d->K * 4u, 1, d->K, (uint32_t)(m.P * d->N), 4, bn);
        } else if (tiles_ok && !(path && !strcmp(path, "naive")) && (m.grouped || d->M % XMR_MMT_BM == 0) && d->N % XMR_MMT_BN == 0 &&
                   d->K % XMR_MMT_BK == 0) {
            variant = "_tiled";
            L.block = xmr_mmt_threads(nc); L.smem = XMR_MMT_SMEM;
            L.ctas = mm_row_tiles(&m, XMR_MMT_BM) * (d->N / XMR_MMT_BN); L.waves = 0;   /* grouped: surplus CTAs exit */
            L.grp_tm = XMR_MMT_BM; L.grp_tiles_n = d->N / XMR_MMT_BN;
        }
        mm_kernel_name(L.name, d->kernel, variant, bt_name, m.grouped, 0, 0, nc, inj);
        break;
    }
    case COAST_K_QSORT:
        if (d->unit_bytes < 4 || (d->unit_bytes & 3u) || d->unit_bytes > 4096u)
            return fail(COAST_ERR_BAD_ARG, "quicksort arrays are 1..1024 int32 (unit_bytes = 4*L, got %u)", d->unit_bytes);
        {   /* two schedulings of the same algorithm (xmr_qsort.cuh): per-unit state machine (default) or nested loops; a ragged
             * batch has the state machine over cost-ordered warp-tiles only (xmr_ragged.cuh) */
            const char* path = getenv("COAST_QSORT_PATH");
            const int nested = path && !strcmp(path, "nested");
            if (ragged && nested)
                return fail(COAST_ERR_UNSUPPORTED, "COAST_QSORT_PATH=nested: ragged quicksort batches (COAST_UNIT_OFFSETS) run the "
                                                   "state-machine scheduling only");
            if (ragged) snprintf(L.name, sizeof L.name, "xmr_qsort_var_inj%d_nc%u", inj, nc);
            else snprintf(L.name, sizeof L.name, "%s_nc%u_inj%d", nested ? "xmr_qsortn" : "xmr_qsort", nc, inj);
        }
        /* one resident wave of persistent warps, each with a private copy of every replica's array, lane-major and CONTIGUOUS
         * per lane (a scan walks one cache line per 32 elements; thread-local memory would put a lane's elements 128 bytes apart) */
        L.block = XMR_QSORT_THREADS; L.waves = 1;
        L.scratch_per_cta = (size_t)XMR_QSORT_THREADS * d->unit_bytes;
        break;
    case COAST_K_CHSTONE_SHA:
        if (d->unit_bytes < 64u || (d->unit_bytes & 63u) || d->unit_bytes >= (1u << 29))
            return fail(COAST_ERR_BAD_ARG, "CHStone sha streams are whole 64-byte blocks, 64 <= unit_bytes < 2^29 (got %u)", d->unit_bytes);
        if (!aligned16 || (((uintptr_t)d->d_out) & 3u)) return fail(COAST_ERR_BAD_ARG, "CHStone sha: d_in must be 16-byte and d_out 4-byte aligned");
        snprintf(L.name, sizeof L.name, "xmr_chsha_nc%u_inj%d", nc, inj);
        break;
    case COAST_K_CHSTONE_AES: {
        const int dec = (d->mode & COAST_AES_DECRYPT) != 0;
        if ((d->mode & COAST_AES_KEY_PER_UNIT) && !d->d_aux) return fail(COAST_ERR_BAD_ARG, "per-unit keys need d_aux");
        if (!aligned16 || (((uintptr_t)d->d_out) & 15u) || ((d->mode & COAST_AES_KEY_PER_UNIT) && (((uintptr_t)d->d_aux) & 15u)))
            return fail(COAST_ERR_BAD_ARG, "CHStone aes buffers must be 16-byte aligned");
        static const char* const stem[2] = { "xmr_chaes_enc", "xmr_chaes_dec" };
        snprintf(L.name, sizeof L.name, "%s_nc%u_inj%d", stem[dec], nc, inj);
        L.block = XMR_AES_THREADS; L.smem = xmr_aes_smem(dec);               /* the same shared-memory tables as the TI kernels */
        break;
    }
    case COAST_K_GEMM_TF32:
    case COAST_K_GEMM_BF16:
    case COAST_K_GEMM_FP8:
    case COAST_K_GEMM_I8:
    case COAST_K_GEMM_F16: {
        /* one body for every operand type (xmr_gemm_tf32.cuh): fp32 operands read as TF32, B^T K-major from a transposing pre-pass
         * into scratch; bfloat16 or float16 operands, 64-element k-blocks and B read in place (no pre-pass, no scratch); or E4M3 or s8
         * operands, 128-element k-blocks and, as for TF32, B^T K-major from a byte-transposing pre-pass (the type's MM_OPS row) */
        const struct mm_op* op = &MM_OPS[d->kernel];
        const unsigned bk = op->bk;
        if (m.grouped && (d->N % xmr_gemm_bn(0) || d->K % bk))
            return fail(COAST_ERR_UNSUPPORTED, "GEMM_%s grouped tiles are 128 x 128 x %u: N must be a multiple of 128 and K of %u "
                                               "(got %u, %u); the products' rows are free", op->ty, bk, bk, d->N, d->K);
        if (!m.grouped && (d->M % XMR_WG_BM || d->N % xmr_gemm_bn(0) || d->K % bk))
            return fail(COAST_ERR_UNSUPPORTED, "GEMM_%s tiles are 128x128x%u: M,N must be multiples of 128 and K of %u (got %u,%u,%u)",
                        op->ty, bk, bk, d->M, d->N, d->K);
        if (!aligned16 || (((uintptr_t)d->d_aux) & 15u) || (((uintptr_t)d->d_out) & 15u)) return fail(COAST_ERR_BAD_ARG, "GEMM buffers must be 16-byte aligned");
        /* unprotected 128 x 256 tiles when N allows (wide), else 128 x 128.  CTA-pair kernels (cluster 2 x 1 x 1,
         * 256-row pair tiles, B multicast) are bit-identical to the single-CTA kernels.  Default: pairs for the unprotected and
         * DWC kernels when the shape allows, the single-CTA kernel for TMR; COAST_GEMM_PAIR=0 / 1 forces one or the other.
         * A batch stacks its products' rows: a pair tile needs the rows of ONE product, so M (per product) % 256 == 0.
         * Groups take 128 x 128 tiles on single CTAs. */
        const int wide = !m.grouped && nc == 1 && d->N % xmr_gemm_bn(1) == 0;
        const char* e = getenv("COAST_GEMM_PAIR");
        const int want_pair = e && (!strcmp(e, "0") || !strcmp(e, "1")) ? e[0] == '1' : nc < 3;
        const int pair = !m.grouped && want_pair && d->M % (2u * XMR_WG_BM) == 0 && d->N % xmr_gemm_bn(nc == 1) == 0 && G.sm_count >= 2;
        /* a caller's B^T is read in place, K-major: BF16 has kernels of its own for it (bt_kernels), TF32, FP8 and I8 only skip the
         * transposing pre-pass */
        mm_kernel_name(L.name, d->kernel, pair ? "p" : nc == 1 && !wide ? "n" : "", m.bt, m.grouped, m.scaled, m.ces == 2, nc, inj);
        { const char* g = getenv("COAST_GEMM_GROUP_M");
          if (g && atoi(g) > 0 && atoi(g) <= (int)XMR_MODE_GROUP_M_MASK) a.mode = (a.mode & ~XMR_MODE_GROUP_M_MASK) | (unsigned)atoi(g); }
        /* L2 eviction priorities: A evict_last, B and C evict_first; COAST_GEMM_L2_HINTS=0 loads and stores with the normal policy */
        { const char* h = getenv("COAST_GEMM_L2_HINTS"); if (!(h && !strcmp(h, "0"))) a.mode |= XMR_MODE_L2_HINTS; }
        /* the unprotected kernel halves the tiles of a short last round; COAST_GEMM_TAIL_SPLIT=0 keeps whole tiles */
        { const char* h = getenv("COAST_GEMM_TAIL_SPLIT"); if (h && !strcmp(h, "0")) a.mode |= XMR_MODE_NO_TAIL_SPLIT; }
        /* persistent CTAs, one per SM (their shared memory allows no second); pairs: an even grid */
        L.block = XMR_WG_THREADS; L.smem = xmr_gemm_smem(wide);
        L.ctas = mm_row_tiles(&m, XMR_WG_BM) * (d->N / xmr_gemm_bn(wide)); L.waves = 1; L.cluster = pair ? 2 : 1;
        L.grp_tm = XMR_WG_BM; L.grp_tiles_n = d->N / xmr_gemm_bn(wide);
        /* B^T of every product into scratch, unless the caller holds it (COAST_MM_B_TRANSPOSED) or BF16 reads B in place */
        const int b_scratch = !op->b_in_place && !m.bt;
        const uintptr_t b_base = b_scratch ? 0 : (uintptr_t)d->d_aux;
        if (b_scratch) {
            L.scratch = (size_t)m.P * d->K * d->N * m.es;
            L.prepass = prepass_transpose_b;
        }
        L.n_maps = 2;
        /* A: the stacked rows of d_in; for groups a placeholder of 128 rows that the scan rebases onto row ro[0] of d_in with R rows
         * (the host does not read the device table).  The placeholder is the B^T scratch, or without it d_aux: d_in of a host-call
         * chunk is biased by ro[first] rows and need not be an address of its own */
        if (m.grouped) plan_wg_map(&L.map[0], op->dt, m.es, b_base, b_scratch, d->K, XMR_WG_BM, 1, XMR_WG_BM);
        else plan_wg_map(&L.map[0], op->dt, m.es, (uintptr_t)d->d_in, 0, d->K, (uint32_t)m.rows, 1, XMR_WG_BM);
        /* B: the stacked B^T, (P N) rows of K, in scratch or the caller's; BF16 without COAST_MM_B_TRANSPOSED: the caller's B,
         * (P K) rows of N in boxes of 64 columns x 64 k-rows */
        plan_wg_map(&L.map[1], op->dt, m.es, b_base, b_scratch, m.b_rows_k ? d->N : d->K, (uint32_t)(m.P * m.b_rows), 1,
                    m.b_rows_k ? XMR_GEMM_BF16_BK : xmr_gemm_b_box(pair));
        break;
    }
    default:
        return fail(COAST_ERR_UNSUPPORTED, "kernel %u is not built into this library yet", d->kernel);
    }
    if (m.grouped && L.grp_tm) {                             /* the group block follows the other scratch */
        L.grp_off = L.scratch;
        L.scratch += (size_t)xmr_mm_grp_bytes(d->M);
    }
    if (ragged) {                                            /* one resident wave pulling cost-ordered warp-tiles (xmr_ragged.cuh) */
        L.waves = 1;
        /* quicksort: the per-warp slots (scratch_per_cta) follow the ragged part in the same allocation */
        L.scratch = (size_t)(d->kernel == COAST_K_QSORT ? xmr_ragged_slots(d->n_units) : xmr_ragged_scratch(d->n_units));
        L.scratch_as_aux = 1;
        L.prepass = prepass_ragged;
    }
    if (!L.ctas) {                                          /* lane-interleaved kernels: each warp takes 32/nc units */
        const uint64_t warps = (d->n_units + upw - 1) / upw, wpc = L.block / 32u;
        L.ctas = (warps + wpc - 1) / wpc;
    }
    return run_plan(&L, d, &a, (CUstream)stream);
}

/* ------------------------------------------------------------------ */
/* counters                                                             */
/* ------------------------------------------------------------------ */
/* Folds the device counters into *out and the reference's globals; *dwc_fired tells the guarded wrappers to call the
 * handler AFTER the single-caller guard is released (a user handler may longjmp or call back into the library). */
static int sync_impl(void* stream, coast_stats* out, int* dwc_fired) {
    int rc = ensure_ctx(); if (rc) return rc;
    if (G.peer_counters) {           /* this GPU's tallies live in the owner's block: wait for the kernels, report nothing */
        DRV(p_cuStreamSynchronize((CUstream)stream));
        if (out) { memset(out, 0, sizeof *out); out->first_fault_unit = ~0ull; }
        if (dwc_fired) *dwc_fired = 0;
        return COAST_OK;
    }
    DRV(p_cuMemcpyDtoHAsync_v2(G.h_counters, G.counters, XMR_CTR_COUNT * sizeof(uint64_t), (CUstream)stream));
    rc = stats_reset_impl(stream); if (rc) return rc;
    DRV(p_cuStreamSynchronize((CUstream)stream));
    coast_stats st;
    st.errors_corrected = G.h_counters[XMR_CTR_ERRORS];
    st.dwc_detected = G.h_counters[XMR_CTR_DWC];
    st.syncs = G.h_counters[XMR_CTR_SYNCS];
    st.injected = G.h_counters[XMR_CTR_INJECTED];
    st.first_fault_unit = G.h_counters[XMR_CTR_FIRST];
    TMR_ERROR_CNT += (uint32_t)st.errors_corrected;          /* i32 wrap, synchronization.cpp:1428-1431 */
    __SYNC_COUNT += st.syncs;
    if (out) *out = st;
    if (dwc_fired) *dwc_fired = st.dwc_detected != 0;
    return COAST_OK;
}
static int sync_guarded(void* stream, coast_stats* out, int call_handler) {
    ENTER();
    int fired = 0, rc = sync_impl(stream, out, &fired);
    leave();
    if (!rc && call_handler && fired) FAULT_DETECTED_DWC();   /* synchronization.cpp:1299-1302 */
    return rc;
}
int coast_sync(void* stream, coast_stats* out) { return sync_guarded(stream, out, 1); }
int coast_sync_noabort(void* stream, coast_stats* out) { return sync_guarded(stream, out, 0); }
int coast_launch(const coast_launch_desc* d, void* stream) { ENTER(); LEAVE(launch_impl(d, stream)); }

/* Multi-GPU counter fold in the kernels themselves (no collective): the owner exports its counter block, the other ranks
 * map it (CUDA IPC, peer access over NVLink) and every later kernel of theirs adds its tallies there with system-scope
 * atomics (Tally::flush).  The owner's coast_sync() then reads the sum over all attached GPUs; the caller orders it after
 * the other ranks' stream synchronisation (a barrier).  An attached rank's coast_sync() waits for its stream and reports zeros. */
int coast_counters_export(void* handle) {
    ENTER();
    int rc = ensure_ctx(); if (rc) LEAVE(rc);
    if (!handle) LEAVE(fail(COAST_ERR_BAD_ARG, "null handle"));
    CUipcMemHandle h;
    CUresult r = p_cuIpcGetMemHandle(&h, G.counters);
    if (r != CUDA_SUCCESS) LEAVE(drv_fail(r, "cuIpcGetMemHandle(counters)"));
    memcpy(handle, &h, sizeof h);
    LEAVE(COAST_OK);
}
int coast_counters_attach(const void* handle) {
    ENTER();
    int rc = ensure_ctx(); if (rc) LEAVE(rc);
    if (!handle) LEAVE(fail(COAST_ERR_BAD_ARG, "null handle"));
    if (G.peer_counters) LEAVE(fail(COAST_ERR_BAD_ARG, "already attached to a peer's counter block (coast_counters_detach first)"));
    CUipcMemHandle h; memcpy(&h, handle, sizeof h);
    CUdeviceptr p = 0;
    CUresult r = p_cuIpcOpenMemHandle_v2(&p, h, CU_IPC_MEM_LAZY_ENABLE_PEER_ACCESS);
    if (r != CUDA_SUCCESS) LEAVE(drv_fail(r, "cuIpcOpenMemHandle(peer counters): no peer access to the owner's GPU?"));
    G.peer_counters = p;
    LEAVE(COAST_OK);
}
int coast_counters_detach(void) {
    ENTER();
    int rc = ensure_ctx(); if (rc) LEAVE(rc);
    if (G.peer_counters) {
        CUresult r = p_cuIpcCloseMemHandle(G.peer_counters);
        G.peer_counters = 0;
        if (r != CUDA_SUCCESS) LEAVE(drv_fail(r, "cuIpcCloseMemHandle(peer counters)"));
    }
    LEAVE(COAST_OK);
}

int coast_stats_snapshot(void* stream, void* d_stats_out) {
    ENTER();
    int rc = ensure_ctx(); if (rc) LEAVE(rc);
    if (!d_stats_out) LEAVE(fail(COAST_ERR_BAD_ARG, "null d_stats_out"));
    CUresult r = p_cuMemcpyDtoDAsync_v2((CUdeviceptr)d_stats_out, G.counters, XMR_CTR_COUNT * sizeof(uint64_t), (CUstream)stream);
    LEAVE(r == CUDA_SUCCESS ? COAST_OK : drv_fail(r, "cuMemcpyDtoDAsync(counters)"));
}

/* ------------------------------------------------------------------ */
/* memory / streams / synthetic data                                    */
/* ------------------------------------------------------------------ */
int coast_malloc(void** p, size_t bytes) { int rc = ensure_ctx(); if (rc) return rc; CUdeviceptr d; DRV(p_cuMemAlloc_v2(&d, bytes ? bytes : 1)); *p = (void*)d; return COAST_OK; }
int coast_free(void* p) { int rc = ensure_ctx(); if (rc) return rc; if (p) DRV(p_cuMemFree_v2((CUdeviceptr)p)); return COAST_OK; }
int coast_memcpy_h2d(void* d, const void* h, size_t n, void* s) { int rc = ensure_ctx(); if (rc) return rc; DRV(p_cuMemcpyHtoDAsync_v2((CUdeviceptr)d, h, n, (CUstream)s)); return COAST_OK; }
int coast_memcpy_d2h(void* h, const void* d, size_t n, void* s) { int rc = ensure_ctx(); if (rc) return rc; DRV(p_cuMemcpyDtoHAsync_v2(h, (CUdeviceptr)d, n, (CUstream)s)); return COAST_OK; }
int coast_memset(void* d, int byte, size_t n, void* s) { int rc = ensure_ctx(); if (rc) return rc; DRV(p_cuMemsetD8Async((CUdeviceptr)d, (unsigned char)byte, n, (CUstream)s)); return COAST_OK; }
int coast_host_alloc(void** h, size_t n) { int rc = ensure_ctx(); if (rc) return rc; DRV(p_cuMemHostAlloc(h, n ? n : 1, 0)); return COAST_OK; }
int coast_host_free(void* h) { int rc = ensure_ctx(); if (rc) return rc; if (h) DRV(p_cuMemFreeHost(h)); return COAST_OK; }
int coast_stream_create(void** s) { int rc = ensure_ctx(); if (rc) return rc; CUstream st; DRV(p_cuStreamCreate(&st, CU_STREAM_NON_BLOCKING)); *s = st; return COAST_OK; }
int coast_stream_destroy(void* s) { int rc = ensure_ctx(); if (rc) return rc; DRV(p_cuStreamDestroy_v2((CUstream)s)); return COAST_OK; }
int coast_stream_sync(void* s) { int rc = ensure_ctx(); if (rc) return rc; DRV(p_cuStreamSynchronize((CUstream)s)); return COAST_OK; }

static int fill_philox_impl(void* d_dst, uint64_t n_words, uint64_t word_base, uint32_t seed, void* stream) {
    int rc = ensure_ctx(); if (rc) return rc;
    if (!n_words) return COAST_OK;
    unsigned long long nw = n_words, wb = word_base;
    void* params[] = { &d_dst, &nw, &wb, &seed };
    uint64_t blks = (n_words + 3) / 4 + 1;
    uint64_t ctas = (blks + 255) / 256, cap = (uint64_t)G.sm_count * 16;
    return launch_small("xmr_fill_philox", (unsigned)(ctas < cap ? ctas : cap), 256, params, (CUstream)stream);
}

/* {clock64, globaltimer ns} per SM into d_out[2 * smid ..] (2 x u64 x SM count, see coast_sm_count()): two probes around a region
 * give the SM clock it really ran at.  Measurement helper of bench.py; not part of the protected path. */
int coast_clock_probe(void* d_out, void* stream) {
    ENTER();
    int rc = ensure_ctx(); if (rc) LEAVE(rc);
    if (!d_out) LEAVE(fail(COAST_ERR_BAD_ARG, "null d_out"));
    void* params[] = { &d_out };
    LEAVE(launch_small("xmr_clock_probe", 4u * (unsigned)G.sm_count, 32, params, (CUstream)stream));
}
int coast_sm_count(void) { return G.inited ? G.sm_count : 0; }

int coast_fill_philox(void* d_dst, uint64_t n_words, uint64_t word_base, uint32_t seed, void* stream) {
    ENTER(); LEAVE(fill_philox_impl(d_dst, n_words, word_base, seed, stream));
}

/* ------------------------------------------------------------------ */
/* host-buffer call: H2D -> xMR kernel -> D2H, chunked over 3 streams    */
/* ------------------------------------------------------------------ */
static int slot_reserve(CUdeviceptr* p, size_t* cap, size_t need) {
    if (*cap >= need) return COAST_OK;
    if (*p) DRV(p_cuMemFree_v2(*p));
    *p = 0; *cap = 0;
    DRV(p_cuMemAlloc_v2(p, need));
    *cap = need;
    return COAST_OK;
}

/* Device-visible alias of a HOST pointer, or 0.  Pinned host memory (cuMemHostAlloc / cudaHostAlloc / cudaHostRegister;
 * torch's pin_memory()) is mapped into the GPU's address space under UVA, so a kernel -- and the TMA unit -- can read and
 * write it over PCIe directly. */
static CUdeviceptr host_alias(const void* h, size_t bytes) {
    if (!h || !bytes) return 0;
    unsigned int mt = 0;
    if (p_cuPointerGetAttribute(&mt, CU_POINTER_ATTRIBUTE_MEMORY_TYPE, (CUdeviceptr)(uintptr_t)h) != CUDA_SUCCESS) return 0;
    if (mt != CU_MEMORYTYPE_HOST) return 0;
    CUdeviceptr d0 = 0, d1 = 0;
    if (p_cuPointerGetAttribute(&d0, CU_POINTER_ATTRIBUTE_DEVICE_POINTER, (CUdeviceptr)(uintptr_t)h) != CUDA_SUCCESS || !d0) return 0;
    /* the last byte must belong to a mapped range too (a view that runs past a registration is not ours to read) */
    if (p_cuPointerGetAttribute(&d1, CU_POINTER_ATTRIBUTE_DEVICE_POINTER, (CUdeviceptr)((uintptr_t)h + bytes - 1)) != CUDA_SUCCESS ||
        d1 != d0 + (bytes - 1)) return 0;
    return d0;
}

/* A host call failed with `rc`: copies of earlier chunks may still be in flight on the caller's buffers, so wait for the three
 * host-call streams before returning -- and keep the error text of the failure, not of the wait. */
static int drain_host_streams(int rc) {
    char keep[sizeof G.err]; memcpy(keep, G.err, sizeof keep);
    for (int i = 0; i < 3; ++i) p_cuStreamSynchronize(G.slot[i].s);
    memcpy(G.err, keep, sizeof keep);
    return rc;
}

/* The chunk pipeline.  A schedule cuts the call into chunks of whole items (units, matmul rows or products); chunk i runs on
 * slot i % 3: its input and aux bytes go up into the slot, its launch reads and writes the slot, its output and status bytes
 * come down, so uploads, kernels and downloads of neighbouring chunks overlap (PCIe is full duplex).  Each chunk is its own
 * launch keyed by the global unit index (unit_base), and the fault plan is keyed by that index, so chunking never changes
 * results. */
typedef struct { uint64_t off, len; } byte_range;           /* bytes [off, off + len) of one of the caller's buffers */
typedef struct {
    uint64_t items;                                          /* items the chunk takes */
    byte_range in, aux, out, stat, rows;                     /* of d_in, d_aux, d_out, d_status and d_rows */
    byte_range sa, sb;                                       /* of d_scale_a and d_scale_b (row-wise scales) */
    uint64_t n_units, unit_base;                             /* of the chunk's launch; unit_base is added to the call's */
    uint32_t M;                                              /* rows of a matmul row block (0: the call's M) */
    uint64_t in_bias, out_bias;                              /* the launch's d_in / d_out are the slot's buffers minus these */
    uint64_t sa_bias;                                        /* ... and its d_scale_a (groups: biased like d_in) */
} host_chunk;

typedef struct host_sched host_sched;
struct host_sched {
    const coast_launch_desc* d;
    /* the chunk after `done` items; *budget is the schedule's running bound (units or bytes), advanced for the next chunk */
    void (*next)(const host_sched* s, uint64_t done, uint64_t* budget, host_chunk* c);
    uint64_t total, budget;                                  /* items of the call; the first chunk's budget */
    uint64_t ib, ab, ob, upi;                                /* per item: bytes of input, aux data and output; units */
    uint64_t min_items, max_items, max_bytes;                /* chunk bounds */
    uint64_t min_in;                                         /* least input slot: an empty input still launches on an address */
    uint64_t shared_b;                                       /* bytes of the matmul's B: uploaded once, every chunk waits for it */
    uint64_t sab, sbb;                                       /* scaled matmuls, per item: bytes of row-wise A and B scales */
    uint64_t shared_sa, shared_sb;                           /* bytes of A and B scales uploaded once with B (tensorwise: 4 and 4) */
    CUdeviceptr zin;                                         /* hybrid: the input's mapped alias, which the kernels read in place */
    int qs, aux_back;                                        /* ragged quicksort (output in place of the input); AES key write-back */
    const char* path;                                        /* what coast_last_host_path() reports */
};

/* Items [first, first + n) of a schedule with fixed bytes per item. */
static void item_chunk(const host_sched* s, uint64_t first, uint64_t n, host_chunk* c) {
    memset(c, 0, sizeof *c);
    c->items = n; c->n_units = n * s->upi; c->unit_base = first * s->upi;
    c->in = (byte_range){ first * s->ib, n * s->ib };
    c->aux = (byte_range){ first * s->ab, n * s->ab };
    c->out = (byte_range){ first * s->ob, n * s->ob };
    c->stat = (byte_range){ c->unit_base, c->n_units };     /* one status byte per unit */
    c->sa = (byte_range){ first * s->sab, n * s->sab };
    c->sb = (byte_range){ first * s->sbb, n * s->sbb };
}

/* Uniform units.  Large chunks amortise the driver work of each chunk, but a fixed size leaves the copy engines idle while the
 * first chunk goes up and the last comes down.  So chunks ramp 1, 2, 4, .. MiB of input up to COAST_HOST_CHUNK_BYTES and
 * shrink again towards the end, each at most half of what remains (tools/e2e_chunk_sweep.py sweeps the bound).  The bounds are
 * in BYTES: a unit larger than the bound (a long CHStone stream, a long SHA message) is a chunk of its own. */
static void next_units(const host_sched* s, uint64_t done, uint64_t* ramp, host_chunk* c) {
    const uint64_t left = s->total - done;
    uint64_t n = *ramp < s->max_items ? *ramp : s->max_items;          /* ramp up */
    if (n > left / 2 && left > 2 * s->min_items) n = left / 2;         /* ramp down */
    if (n < s->min_items) n = s->min_items;
    if (n > left) n = left;
    *ramp *= 2;
    item_chunk(s, done, n, c);
}

/* Ragged units (COAST_UNIT_OFFSETS, d_aux = the caller's host offsets): a chunk is the longest unit range whose bytes
 * [off[first], off[end]) -- counted twice for quicksort, in and out -- and per-unit offset and output bytes fit the budget,
 * which ramps 1, 2, 4, .. MiB up to COAST_HOST_CHUNK_BYTES; a longer unit is a chunk of its own.  The chunk uploads its bytes
 * and its offset slice off[first .. end] unchanged and launches with the slot's address minus off[first] as d_in (exact under
 * u64 wraparound), so the caller's offsets are never rewritten.  Quicksort sorts each array in place of its input bytes: the
 * output is the same span, downloaded from an output slot biased the same way. */
static void next_ragged(const host_sched* s, uint64_t first, uint64_t* budget, host_chunk* c) {
    const uint64_t* off = (const uint64_t*)s->d->d_aux;
    const uint64_t per_unit = s->ob + 8u, span_copies = s->qs ? 2u : 1u;
    uint64_t e = first + 1;
    while (e < s->total && (off[e + 1] - off[first]) * span_copies + (e + 1 - first) * per_unit <= *budget) ++e;
    *budget = *budget * 2 < s->max_bytes ? *budget * 2 : s->max_bytes;
    memset(c, 0, sizeof *c);
    c->items = c->n_units = e - first; c->unit_base = first;
    c->in = (byte_range){ off[first], off[e] - off[first] }; c->in_bias = off[first];
    c->aux = (byte_range){ first * 8u, (e - first + 1) * 8u };
    c->out = s->qs ? c->in : (byte_range){ first * s->ob, (e - first) * s->ob };
    c->out_bias = s->qs ? off[first] : 0;
    c->stat = (byte_range){ first, e - first };
}

/* Batched matmuls (COAST_MM_BATCHED): chunks of max_items whole products, each with its own A, B and C. */
static void next_products(const host_sched* s, uint64_t done, uint64_t* budget, host_chunk* c) {
    (void)budget;
    const uint64_t left = s->total - done;
    item_chunk(s, done, left < s->max_items ? left : s->max_items, c);
}

/* Grouped matmuls (COAST_MM_GROUPED, d_rows = the caller's host row offsets ro[]; ib, ab and ob are the bytes of a row of A, of
 * one product's B and of a row of C): a chunk is the longest run of whole products whose A rows, B matrices, C rows and offsets
 * fit COAST_HOST_CHUNK_BYTES; a larger product is a chunk of its own.  The chunk
 * uploads its offset slice ro[first .. end] unchanged and launches with the slots' addresses minus ro[first] rows as d_in and
 * d_out (exact under u64 wraparound, as next_ragged), so the caller's offsets are never rewritten. */
static void next_groups(const host_sched* s, uint64_t first, uint64_t* budget, host_chunk* c) {
    const uint64_t* ro = (const uint64_t*)s->d->d_rows;
    const uint64_t N = s->d->N;
    uint64_t e = first + 1;
    while (e < s->total && (ro[e + 1] - ro[first]) * (s->ib + s->ob) + (e + 1 - first) * (s->ab + 8u) + 8u <= *budget) ++e;
    memset(c, 0, sizeof *c);
    const uint64_t rows = ro[e] - ro[first];
    c->items = e - first; c->M = (uint32_t)(e - first);
    c->n_units = rows * N; c->unit_base = (ro[first] - ro[0]) * N;
    c->in = (byte_range){ ro[first] * s->ib, rows * s->ib }; c->in_bias = ro[first] * s->ib;
    c->aux = (byte_range){ first * s->ab, (e - first) * s->ab };
    c->out = (byte_range){ ro[first] * s->ob, rows * s->ob }; c->out_bias = ro[first] * s->ob;
    c->rows = (byte_range){ first * 8u, (e - first + 1) * 8u };
    c->sa = (byte_range){ ro[first] * s->sab, rows * s->sab }; c->sa_bias = ro[first] * s->sab;
    c->sb = (byte_range){ first * s->sbb, (e - first) * s->sbb };
}

/* Matmul row blocks: max_items rows of A up and of C down per chunk; B is the schedule's shared operand. */
static void next_row_block(const host_sched* s, uint64_t done, uint64_t* budget, host_chunk* c) {
    next_products(s, done, budget, c);
    c->M = (uint32_t)c->items;
}

static void grow(uint64_t* need, uint64_t len) { if (len > *need) *need = len; }
static uint64_t align16(uint64_t x) { return (x + 15u) & ~(uint64_t)15u; }

/* Runs a call's chunks.  The schedule is walked twice: once to size each slot for the largest chunk it gets -- every slot is
 * reserved before the first copy, so a failed allocation never leaves a partly written output -- and once to run. */
static int run_chunks(const host_sched* s, coast_stats* out, int* dwc_fired) {
    const coast_launch_desc* d = s->d;
    struct { uint64_t in, aux, out, stat, rows, sc; } need[3];
    memset(need, 0, sizeof need);
    uint64_t n_chunks = 0;
    for (uint64_t done = 0, budget = s->budget; done < s->total; ++n_chunks) {
        host_chunk c; s->next(s, done, &budget, &c);
        const int i = (int)(n_chunks % 3);
        grow(&need[i].in, c.in.len); grow(&need[i].aux, c.aux.len); grow(&need[i].out, c.out.len); grow(&need[i].stat, c.stat.len);
        grow(&need[i].rows, c.rows.len); grow(&need[i].sc, align16(c.sa.len) + c.sb.len);
        done += c.items;
    }
    int rc;
    for (int i = 0; i < 3 && (uint64_t)i < n_chunks; ++i) {
        host_slot* sl = &G.slot[i];
        const uint64_t in = need[i].in > s->min_in ? need[i].in : s->min_in;
        if (!s->zin && (rc = slot_reserve(&sl->in.p, &sl->in.cap, in))) return rc;
        if ((rc = slot_reserve(&sl->out.p, &sl->out.cap, s->qs ? in : need[i].out))) return rc;   /* quicksort: in's twin */
        if ((rc = slot_reserve(&sl->aux.p, &sl->aux.cap, need[i].aux))) return rc;
        if (d->d_status && (rc = slot_reserve(&sl->stat.p, &sl->stat.cap, need[i].stat))) return rc;
        if (need[i].rows && (rc = slot_reserve(&sl->rows.p, &sl->rows.cap, need[i].rows))) return rc;
        if (need[i].sc && (rc = slot_reserve(&sl->sc.p, &sl->sc.cap, need[i].sc))) return rc;
    }
    /* what every chunk shares goes up once: [B][A's scales][B's scales], each part 16-byte aligned */
    const uint64_t sa_at = align16(s->shared_b), sb_at = sa_at + align16(s->shared_sa);
    const int shared = s->shared_b || s->shared_sa || s->shared_sb;
    if (shared) {
        if ((rc = slot_reserve(&G.h_b.p, &G.h_b.cap, s->shared_sa || s->shared_sb ? sb_at + s->shared_sb : s->shared_b))) return rc;
        if (!G.ev_b) DRV(p_cuEventCreate(&G.ev_b, CU_EVENT_DISABLE_TIMING));
    }
#define STEP(call) do { CUresult r_ = (call); if (r_ != CUDA_SUCCESS) { rc = drv_fail(r_, #call); goto fail; } } while (0)
    uint64_t done = 0, budget = s->budget;
    for (uint64_t i = 0; done < s->total; ++i) {
        host_chunk k; s->next(s, done, &budget, &k);
        const host_slot* sl = &G.slot[i % 3];
        coast_launch_desc c = *d;
        if (s->zin) {
            c.d_in = (const void*)(uintptr_t)(s->zin + k.in.off);
        } else {
            if (k.in.len) STEP(p_cuMemcpyHtoDAsync_v2(sl->in.p, (const uint8_t*)d->d_in + k.in.off, (size_t)k.in.len, sl->s));
            c.d_in = (const void*)(uintptr_t)(sl->in.p - k.in_bias);
        }
        if (k.aux.len) {
            STEP(p_cuMemcpyHtoDAsync_v2(sl->aux.p, (const uint8_t*)d->d_aux + k.aux.off, (size_t)k.aux.len, sl->s));
            c.d_aux = (const void*)sl->aux.p;
        }
        if (k.rows.len) {
            STEP(p_cuMemcpyHtoDAsync_v2(sl->rows.p, (const uint8_t*)d->d_rows + k.rows.off, (size_t)k.rows.len, sl->s));
            c.d_rows = (const void*)sl->rows.p;
        }
        if (k.sa.len || k.sb.len) {                          /* row-wise scales of the chunk's rows and products */
            const CUdeviceptr sbp = sl->sc.p + align16(k.sa.len);
            if (k.sa.len) STEP(p_cuMemcpyHtoDAsync_v2(sl->sc.p, (const uint8_t*)d->d_scale_a + k.sa.off, (size_t)k.sa.len, sl->s));
            if (k.sb.len) STEP(p_cuMemcpyHtoDAsync_v2(sbp, (const uint8_t*)d->d_scale_b + k.sb.off, (size_t)k.sb.len, sl->s));
            if (k.sa.len) c.d_scale_a = (const void*)(uintptr_t)(sl->sc.p - k.sa_bias);
            if (k.sb.len) c.d_scale_b = (const void*)(uintptr_t)sbp;
        }
        if (shared) {                                        /* B (and shared scales) follow the first chunk's input, on stream 1 */
            if (i == 0) {
                if (s->shared_b) STEP(p_cuMemcpyHtoDAsync_v2(G.h_b.p, d->d_aux, (size_t)s->shared_b, G.slot[1].s));
                if (s->shared_sa) STEP(p_cuMemcpyHtoDAsync_v2(G.h_b.p + sa_at, d->d_scale_a, (size_t)s->shared_sa, G.slot[1].s));
                if (s->shared_sb) STEP(p_cuMemcpyHtoDAsync_v2(G.h_b.p + sb_at, d->d_scale_b, (size_t)s->shared_sb, G.slot[1].s));
                STEP(p_cuEventRecord(G.ev_b, G.slot[1].s));
            }
            STEP(p_cuStreamWaitEvent(sl->s, G.ev_b, 0));
            if (s->shared_b) c.d_aux = (const void*)G.h_b.p;
            if (s->shared_sa) c.d_scale_a = (const void*)(uintptr_t)(G.h_b.p + sa_at);
            if (s->shared_sb) c.d_scale_b = (const void*)(uintptr_t)(G.h_b.p + sb_at);
        }
        c.d_out = (void*)(uintptr_t)(sl->out.p - k.out_bias);
        if (d->d_status) c.d_status = (void*)sl->stat.p;    /* kernels index status[] chunk-locally */
        c.n_units = k.n_units; c.unit_base = d->unit_base + k.unit_base;
        if (k.M) c.M = k.M;
        rc = launch_impl(&c, sl->s); if (rc) goto fail;
        if (k.out.len) STEP(p_cuMemcpyDtoHAsync_v2((uint8_t*)d->d_out + k.out.off, sl->out.p, (size_t)k.out.len, sl->s));
        if (s->aux_back) STEP(p_cuMemcpyDtoHAsync_v2((uint8_t*)d->d_aux + k.aux.off, sl->aux.p, (size_t)k.aux.len, sl->s));
        if (d->d_status) STEP(p_cuMemcpyDtoHAsync_v2((uint8_t*)d->d_status + k.stat.off, sl->stat.p, (size_t)k.stat.len, sl->s));
        done += k.items;
    }
#undef STEP
    G.last_host_path = s->path;
    DRV(p_cuStreamSynchronize(G.slot[0].s)); DRV(p_cuStreamSynchronize(G.slot[1].s));
    return sync_impl(G.slot[2].s, out, dwc_fired);
fail:
    return drain_host_streams(rc);
}

/* `d_in` / `d_out` / `d_aux` / `d_status` of the descriptor are HOST pointers here.  The policy of the host call: the refusals,
 * which schedule cuts the call into chunks and, for the uniform kernels, whether the bytes move by staged copies, hybrid or one
 * zero-copy launch. */
static int run_host_impl(const coast_launch_desc* d, coast_stats* out, int* dwc_fired) {
    int rc = ensure_ctx(); if (rc) return rc;
    if (!d) return fail(COAST_ERR_BAD_ARG, "null descriptor");
    if (d->plan && d->plan->mode == COAST_PLAN_TABLE) return fail(COAST_ERR_UNSUPPORTED, "coast_run_host: TABLE plans need device pointers; use coast_launch");
    for (int i = 0; i < 3; ++i) if (!G.slot[i].s) DRV(p_cuStreamCreate(&G.slot[i].s, CU_STREAM_NON_BLOCKING));
    const char* hp = getenv("COAST_HOST_PATH");
    uint64_t chunk_bytes = 16ull << 20;                      /* largest chunk (tuning knob; ragged and batched: of all its bytes) */
    { const char* e = getenv("COAST_HOST_CHUNK_BYTES"); if (e && atoll(e) > 0) chunk_bytes = (uint64_t)atoll(e); }
    host_sched s; memset(&s, 0, sizeof s);
    s.d = d; s.upi = 1; s.path = "staged";
    if ((rc = mm_bit_refused(d, COAST_MM_B_TRANSPOSED)) || (rc = mm_scale_check(d)) || (rc = mm_out_check(d))) return rc;

    if (d->mode & COAST_UNIT_OFFSETS) {                      /* ragged: staged only */
        if ((rc = ragged_check(d))) return rc;
        if (hp && (!strcmp(hp, "zerocopy") || !strcmp(hp, "hybrid")))
            return fail(COAST_ERR_UNSUPPORTED, "COAST_HOST_PATH=%s: ragged host calls (COAST_UNIT_OFFSETS) are staged only", hp);
        if (d->n_units == 0) return sync_impl(G.slot[2].s, out, dwc_fired);
        if (!d->d_in || !d->d_out) return fail(COAST_ERR_BAD_ARG, "null host buffer");
        const uint64_t* off = (const uint64_t*)d->d_aux, n = d->n_units;
        s.qs = d->kernel == COAST_K_QSORT;
        for (uint64_t u = 0; u < n; ++u)
            if (off[u + 1] < off[u] || off[u + 1] - off[u] > d->unit_bytes)
                return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: unit %llu runs from offset %llu to %llu; offsets must not decrease and no "
                                               "length may exceed unit_bytes (%u)", (unsigned long long)u, (unsigned long long)off[u],
                            (unsigned long long)off[u + 1], d->unit_bytes);
        if (s.qs)
            for (uint64_t u = 0; u <= n; ++u)
                if (off[u] & 3u)
                    return fail(COAST_ERR_BAD_ARG, "COAST_UNIT_OFFSETS: offset %llu is %llu; quicksort offsets must be multiples of 4",
                                (unsigned long long)u, (unsigned long long)off[u]);
        s.next = next_ragged; s.total = n; s.ob = KINFO[d->kernel].out_bytes; s.min_in = 16;
        s.budget = (1ull << 20) < chunk_bytes ? (1ull << 20) : chunk_bytes; s.max_bytes = chunk_bytes;
        return run_chunks(&s, out, dwc_fired);
    }
    mm_shape m;
    if ((rc = mm_check(d, &m))) return rc;
    if (is_matmul(d->kernel)) {
        if (d->d_status) return fail(COAST_ERR_UNSUPPORTED, "coast_run_host: d_status is not staged for the matmul kernels; use coast_launch");
        const uint64_t a_row = (uint64_t)d->K * m.es, c_row = (uint64_t)d->N * m.ces, bb = (uint64_t)d->K * d->N * m.es;
        if (m.grouped) {                                     /* whole products per chunk, the offsets checked first */
            const uint64_t* ro = (const uint64_t*)d->d_rows;
            for (uint32_t g = 0; g < d->M; ++g)
                if (ro[g + 1] < ro[g])
                    return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: product %u runs from row %llu to %llu; row offsets must not decrease",
                                g, (unsigned long long)ro[g], (unsigned long long)ro[g + 1]);
            if (ro[d->M] - ro[0] != m.rows)
                return fail(COAST_ERR_BAD_ARG, "COAST_MM_GROUPED: the products hold %llu rows but n_units / N is %llu",
                            (unsigned long long)(ro[d->M] - ro[0]), (unsigned long long)m.rows);
            if (m.rows && (!d->d_in || !d->d_out || !d->d_aux)) return fail(COAST_ERR_BAD_ARG, "null host buffer");
            s.next = next_groups; s.total = m.P; s.ib = a_row; s.ab = bb; s.ob = c_row;
            s.max_bytes = chunk_bytes; s.budget = chunk_bytes; s.min_in = 16; s.path = "groups";
        } else if (m.batched) {                              /* as many whole products as the chunk bytes hold, at least one */
            if (!d->d_in || !d->d_out || !d->d_aux) return fail(COAST_ERR_BAD_ARG, "null host buffer");
            s.next = next_products; s.total = m.P; s.upi = (uint64_t)d->M * d->N;
            s.ib = d->M * a_row; s.ab = bb; s.ob = d->M * c_row;
            s.max_items = chunk_bytes / (s.ib + s.ab + s.ob) ? chunk_bytes / (s.ib + s.ab + s.ob) : 1u;
        } else {
            /* B (the replicated operand) goes up once; C comes in at most 8 blocks of whole 128-row groups.  Small or oddly
             * shaped problems go in one block. */
            uint64_t rows = d->M;
            if (d->M % 128u == 0 && d->M >= 512u && !(hp && !strcmp(hp, "one-shot"))) {
                const uint64_t blocks = d->M / 128u < 8u ? d->M / 128u : 8u;
                rows = ((d->M / 128u + blocks - 1u) / blocks) * 128u;
            }
            s.next = next_row_block; s.total = d->M; s.upi = d->N; s.ib = a_row; s.ob = c_row;
            s.max_items = rows; s.shared_b = bb;
            s.path = rows < d->M ? "row-blocks" : "one-shot";
        }
        /* scales: tensorwise, the two floats go up once; row-wise, each chunk takes the A scales of its rows and the B scales of its
         * products, except that row blocks share B and so share its scales.  The chunks are those of the unscaled call. */
        if (m.scaled && !m.rowwise) { s.shared_sa = 4; s.shared_sb = 4; }
        if (m.rowwise) {
            s.sab = 4u * (m.batched ? d->M : 1u);
            if (m.grouped || m.batched) s.sbb = 4ull * d->N;
            else s.shared_sb = 4ull * d->N;
        }
        return run_chunks(&s, out, dwc_fired);
    }
    const uint64_t ob = coast_out_bytes(d->kernel, d->unit_bytes), ib = in_bytes_per_unit(d);
    /* a zero-length SHA-256 message (sha256_hash(len = 0) hashes one padded block) has nothing to stage */
    if (!ob || (!ib && d->kernel != COAST_K_SHA256)) return fail(COAST_ERR_UNSUPPORTED, "coast_run_host: kernel %u", d->kernel);
    const int per_unit_key = aux_bytes_per_unit(d) != 0;
    if (d->n_units == 0) return sync_impl(G.slot[2].s, out, dwc_fired);

    /* Three ways to move the bytes (COAST_HOST_PATH=staged|hybrid|zerocopy overrides the default):
     *   staged  : H2D -> kernel -> D2H per chunk over three streams (any host memory);
     *   hybrid  : pinned input + a kernel that reads each input byte once: the chunks' kernels read mapped host memory
     *             directly through the TMA ring (no upload copies, no input staging), outputs are staged and downloaded
     *             per chunk;
     *   zerocopy: ONE launch reads and WRITES mapped host memory: SM stores of 16-32 bytes per lane to host memory
     *             are small PCIe writes, so it is meant for calls whose output is small. */
    const int streams_once = KINFO[d->kernel].streams_once;
    /* default: staged -- except when the output is tiny next to the input (crc16: 2 of 64 bytes, CHStone sha: 20 bytes per
     * stream), where one zero-copy launch on pinned buffers reads each input byte once and saves the chunk pipeline's copies */
    const int tiny_out = ob * 8u <= ib;
    const int want = hp ? (!strcmp(hp, "zerocopy") ? 2 : !strcmp(hp, "hybrid") ? 1 : 0) : (tiny_out ? 2 : G.host_path_default);
    CUdeviceptr zin = 0;
    if (streams_once && want && ib) zin = host_alias(d->d_in, (size_t)(d->n_units * ib));
    if (want == 2 && streams_once) {
        CUdeviceptr zi = ib ? zin : (CUdeviceptr)G.counters /* never read */;
        CUdeviceptr zo = host_alias(d->d_out, (size_t)(d->n_units * ob));
        CUdeviceptr za = per_unit_key ? host_alias(d->d_aux, (size_t)(d->n_units * aux_bytes_per_unit(d))) : 0;
        CUdeviceptr zs = d->d_status ? host_alias(d->d_status, (size_t)d->n_units) : 0;
        if (zi && zo && (!per_unit_key || za) && (!d->d_status || zs)) {
            coast_launch_desc c = *d;
            c.d_in = (void*)zi; c.d_out = (void*)zo;
            if (per_unit_key) c.d_aux = (void*)za;
            if (d->d_status) c.d_status = (void*)zs;
            rc = launch_impl(&c, G.slot[2].s); if (rc) return rc;
            G.last_host_path = "zerocopy";
            return sync_impl(G.slot[2].s, out, dwc_fired);
        }
        if (hp) return fail(COAST_ERR_BAD_ARG, "COAST_HOST_PATH=zerocopy needs pinned (mapped) host buffers");
        zin = 0;                                                   /* the default policy falls back to staged copies for pageable memory */
    }
    if (hp && want == 1 && streams_once && ib && !zin) return fail(COAST_ERR_BAD_ARG, "COAST_HOST_PATH=hybrid needs a pinned (mapped) input buffer");
    const uint64_t ibs = ib ? ib : 1;                              /* divisor of the chunk bounds */
    s.next = next_units; s.total = d->n_units; s.ib = ib; s.ab = aux_bytes_per_unit(d); s.ob = ob; s.min_in = 16;
    s.min_items = (1ull << 20) / ibs > 1u ? (1ull << 20) / ibs : 1u;
    s.max_items = chunk_bytes / ibs > s.min_items ? chunk_bytes / ibs : s.min_items;
    s.budget = s.min_items;
    s.aux_back = per_unit_key && d->kernel == COAST_K_AES128 && (d->mode & COAST_AES_KEY_WRITEBACK);
    s.zin = zin;                                                   /* nonzero only when hybrid was asked for */
    if (zin) s.path = "hybrid";
    return run_chunks(&s, out, dwc_fired);
}
static int run_host_guarded(const coast_launch_desc* d, coast_stats* out, int call_handler) {
    ENTER();
    int fired = 0, rc = run_host_impl(d, out, &fired);
    leave();
    if (!rc && call_handler && fired) FAULT_DETECTED_DWC();   /* synchronization.cpp:1299-1302 */
    return rc;
}
const char* coast_last_host_path(void) { return G.last_host_path ? G.last_host_path : ""; }
int coast_run_host(const coast_launch_desc* d, coast_stats* out) { return run_host_guarded(d, out, 1); }
int coast_run_host_noabort(const coast_launch_desc* d, coast_stats* out) { return run_host_guarded(d, out, 0); }

/* ------------------------------------------------------------------ */
/* the four reference entry points (what the unchanged tests call)      */
/* ------------------------------------------------------------------ */
static void entry_mode(uint32_t* nc, uint32_t* fl) {
    if (!G.inited) {
        const char* dv = getenv("COAST_DEVICE");
        int rc = coast_init(dv ? atoi(dv) : 0);
        if (rc) { fprintf(stderr, "coast_rt: cannot run the protected region on a GPU: %s\n", G.err); abort(); }
    }
    if (!G.def_set) { const char* env = getenv("COAST_OPT_PASSES"); coast_set_opt_passes(env ? env : ""); }
    *nc = G.def_nc; *fl = G.def_flags;
}
static void entry_run(coast_launch_desc* d) {
    int rc = coast_run_host(d, NULL);
    if (rc) { fprintf(stderr, "coast_rt: protected launch failed: %s\n", G.err); abort(); }
}

unsigned short coast_xmr_crc16(const unsigned char* data_p, unsigned char length) {
    coast_launch_desc d; memset(&d, 0, sizeof d);
    entry_mode(&d.num_clones, &d.flags);
    unsigned short out = 0xFFFF;                               /* crc of the empty message (crc16.c:23) */
    if (!length) return out;
    d.kernel = COAST_K_CRC16; d.n_units = 1; d.unit_bytes = length; d.d_in = data_p; d.d_out = &out;
    entry_run(&d);
    return out;
}
void coast_xmr_sha256_hash(unsigned char ctx_data[], uint32_t ctx_bitlen[], uint32_t ctx_state[], unsigned char data[],
                           uint32_t len, unsigned char hash[]) {
    coast_launch_desc d; memset(&d, 0, sizeof d);
    entry_mode(&d.num_clones, &d.flags);
    unsigned char dummy = 0;
    d.kernel = COAST_K_SHA256; d.n_units = 1; d.unit_bytes = len; d.d_in = len ? data : &dummy; d.d_out = hash;
    entry_run(&d);
    /* The caller-visible scratch the reference leaves behind (sha256_common_tmr.c:101-180): replicas keep it in registers,
     * so it is rebuilt here from the voted digest and the message -- marshalling, not computation.
     *   ctx_state : the final chaining value = the digest words, big-endian (:169-178)
     *   ctx_bitlen: {low, high} of 8*len (DBL_INT_ADD, :124,155)
     *   ctx_data  : the last block fed to sha256_transform (:132-163) */
    if (ctx_state)
        for (int i = 0; i < 8; ++i)
            ctx_state[i] = ((uint32_t)hash[4 * i] << 24) | ((uint32_t)hash[4 * i + 1] << 16) | ((uint32_t)hash[4 * i + 2] << 8) | hash[4 * i + 3];
    const uint32_t lo = len << 3, hi = len >> 29;
    if (ctx_bitlen) { ctx_bitlen[0] = lo; ctx_bitlen[1] = hi; }
    if (ctx_data) {
        const uint32_t rem = len & 63u;
        if (rem < 56u) {
            memcpy(ctx_data, data + (len - rem), rem);
            ctx_data[rem] = 0x80; memset(ctx_data + rem + 1, 0, 55u - rem);
        } else {
            memset(ctx_data, 0, 56);                               /* the extra block: sha_memset(ctx_data, 0, 56) :142-150 */
        }
        ctx_data[63] = (unsigned char)lo; ctx_data[62] = (unsigned char)(lo >> 8); ctx_data[61] = (unsigned char)(lo >> 16); ctx_data[60] = (unsigned char)(lo >> 24);
        ctx_data[59] = (unsigned char)hi; ctx_data[58] = (unsigned char)(hi >> 8); ctx_data[57] = (unsigned char)(hi >> 16); ctx_data[56] = (unsigned char)(hi >> 24);
    }
}
void coast_xmr_aes_enc_dec(unsigned char* state, unsigned char* key, unsigned char dir) {
    coast_launch_desc d; memset(&d, 0, sizeof d);
    entry_mode(&d.num_clones, &d.flags);
    /* per-unit-key mode with write-back so key[] is mutated exactly as TI_aes_128.c:107-231 does */
    d.kernel = COAST_K_AES128; d.n_units = 1; d.d_in = state; d.d_out = state; d.d_aux = key;
    d.mode = (dir ? COAST_AES_DECRYPT : 0) | COAST_AES_KEY_PER_UNIT | COAST_AES_KEY_WRITEBACK;
    entry_run(&d);
}
void coast_xmr_chstone_sha_stream(const unsigned char* indata, const int* in_i, int vsize, int block_size, uint32_t* digest) {
    /* sha_stream (sha.c:182-193) feeds chunk j = indata[j][0 .. in_i[j]) to sha_update; with whole-block chunks that is the
     * hash of the concatenation, which is what one unit of the kernel computes */
    size_t total = 0;
    for (int j = 0; j < vsize; ++j) {
        if (in_i[j] < 0 || in_i[j] > block_size || (in_i[j] & 63)) {
            fprintf(stderr, "coast_rt: sha_stream chunk %d has %d bytes; only whole 64-byte blocks are supported\n", j, in_i[j]);
            abort();
        }
        total += (size_t)in_i[j];
    }
    unsigned char* cat = (unsigned char*)malloc(total ? total : 1);
    if (!cat) abort();
    size_t off = 0;
    for (int j = 0; j < vsize; ++j) { memcpy(cat + off, indata + (size_t)j * (size_t)block_size, (size_t)in_i[j]); off += (size_t)in_i[j]; }
    coast_launch_desc d; memset(&d, 0, sizeof d);
    entry_mode(&d.num_clones, &d.flags);
    d.kernel = COAST_K_CHSTONE_SHA; d.n_units = 1; d.unit_bytes = (uint32_t)total; d.d_in = cat; d.d_out = digest;
    entry_run(&d);
    free(cat);
}
void coast_xmr_chstone_aes(int* statemt, const int* key, int type, int dir) {
    if (type != 128128) {
        fprintf(stderr, "coast_rt: chstone/aes type %d: only 128128 (the benchmark's, aes.c:126-127) has a protected kernel\n", type);
        abort();
    }
    coast_launch_desc d; memset(&d, 0, sizeof d);
    entry_mode(&d.num_clones, &d.flags);
    /* 16-byte aligned bounce buffers: the program's statemt[] / key[] are plain int arrays */
    int st[16] __attribute__((aligned(16))), k[16] __attribute__((aligned(16)));
    memcpy(st, statemt, sizeof st); memcpy(k, key, sizeof k);
    d.kernel = COAST_K_CHSTONE_AES; d.n_units = 1; d.d_in = st; d.d_out = st; d.d_aux = k;
    d.mode = (dir ? COAST_AES_DECRYPT : 0) | COAST_AES_KEY_PER_UNIT;
    entry_run(&d);
    memcpy(statemt, st, sizeof st);
}
void coast_xmr_matrix_multiply_u32(const uint32_t* f, const uint32_t* s, uint32_t* r, int side) {
    coast_launch_desc d; memset(&d, 0, sizeof d);
    entry_mode(&d.num_clones, &d.flags);
    d.kernel = COAST_K_MM_U32; d.M = d.N = d.K = (uint32_t)side; d.n_units = (uint64_t)side * side;
    d.d_in = f; d.d_aux = s; d.d_out = r;
    entry_run(&d);
}
