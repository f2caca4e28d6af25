/*
 * mock_cuda.c -- a stand-in for libcuda.so.1 that lets the HOST logic of libcoast_rt.so run on a GPU-less box.
 *
 * TEST INFRASTRUCTURE ONLY (tests/mock_run.py builds it into a temp dir and puts that dir on LD_LIBRARY_PATH of a
 * child process).  It executes NO workload: kernels are recorded, not run.  What it does check, the way the real driver
 * would fail: every copy stays inside a live allocation, launch geometry and dynamic shared memory are within sm_90
 * limits, tensor maps obey the cuTensorMapEncodeTiled constraints for their element type (UINT8, BFLOAT16, UINT32,
 * FLOAT32), nothing leaks at exit.  Every call that matters is appended as one JSON line to $MOCK_CUDA_LOG.
 */
#include <cuda.h>
#include <elf.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define MAX_ALLOC 4096
static struct { uintptr_t base; size_t size; int live; int host; } allocs[MAX_ALLOC];
static int n_allocs;
static FILE* logf;
static int fake_ctx, fake_mod;
typedef struct { char name[96]; int max_dyn_smem; } mock_fn;
static mock_fn fns[512];
static int n_fns;
static int n_streams;

static void log_open(void) {
    if (logf) return;
    const char* p = getenv("MOCK_CUDA_LOG");
    logf = p ? fopen(p, "a") : NULL;
}
#define LOG(...) do { log_open(); if (logf) { fprintf(logf, __VA_ARGS__); fputc('\n', logf); fflush(logf); } } while (0)

static CUresult bad(const char* what) { LOG("{\"op\":\"error\",\"what\":\"%s\"}", what); return CUDA_ERROR_INVALID_VALUE; }

static int find_alloc(uintptr_t p, size_t n) {
    for (int i = 0; i < n_allocs; ++i)
        if (allocs[i].live && p >= allocs[i].base && p + n <= allocs[i].base + allocs[i].size) return i;
    return -1;
}
static CUresult do_alloc(CUdeviceptr* out, size_t n, int host) {
    if (!n || n_allocs >= MAX_ALLOC) return CUDA_ERROR_INVALID_VALUE;
    const char* fa = getenv("MOCK_CUDA_FAIL_ALLOC_AFTER");              /* fault injection: the k-th allocation and later ones fail */
    if (fa && n_allocs >= atoi(fa)) return CUDA_ERROR_OUT_OF_MEMORY;
    if (n > ((size_t)6 << 30)) return CUDA_ERROR_OUT_OF_MEMORY;          /* the box is small: huge requests fail like OOM */
    void* p = NULL;
    if (posix_memalign(&p, 512, n)) return CUDA_ERROR_OUT_OF_MEMORY;      /* cuMemAlloc returns >= 256-byte aligned memory */
    allocs[n_allocs].base = (uintptr_t)p; allocs[n_allocs].size = n; allocs[n_allocs].live = 1; allocs[n_allocs].host = host;
    LOG("{\"op\":\"alloc\",\"id\":%d,\"bytes\":%zu,\"host\":%d,\"ptr\":%llu}", n_allocs, n, host, (unsigned long long)(uintptr_t)p);
    n_allocs++;
    *out = (CUdeviceptr)(uintptr_t)p;
    return CUDA_SUCCESS;
}
static CUresult do_free(CUdeviceptr d) {
    for (int i = 0; i < n_allocs; ++i)
        if (allocs[i].live && allocs[i].base == (uintptr_t)d) {
            allocs[i].live = 0; free((void*)allocs[i].base);
            LOG("{\"op\":\"free\",\"id\":%d}", i);
            return CUDA_SUCCESS;
        }
    return bad("free of an unknown pointer");
}
__attribute__((destructor)) static void report_leaks(void) {
    int live = 0; for (int i = 0; i < n_allocs; ++i) live += allocs[i].live;
    LOG("{\"op\":\"exit\",\"live_allocations\":%d}", live);
}

CUresult cuInit(unsigned int f) { (void)f; return CUDA_SUCCESS; }
CUresult cuDeviceGet(CUdevice* d, int ord) { if (ord != 0) return CUDA_ERROR_INVALID_DEVICE; *d = 0; return CUDA_SUCCESS; }
CUresult cuDeviceGetAttribute(int* v, CUdevice_attribute a, CUdevice d) {
    (void)d;
    switch (a) {
    case CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR: *v = getenv("MOCK_CUDA_CC_MAJOR") ? atoi(getenv("MOCK_CUDA_CC_MAJOR")) : 9; break;
    case CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR: *v = 0; break;
    case CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT: *v = 132; break;
    default: *v = 0;
    }
    return CUDA_SUCCESS;
}
CUresult cuDeviceGetPCIBusId(char* s, int len, CUdevice d) { (void)d; snprintf(s, (size_t)len, "0000:FF:1F.7"); return CUDA_SUCCESS; }   /* no such sysfs node: NUMA binding is skipped */
/* pinned host allocations are "mapped": their device alias is the pointer itself; anything else is unknown to the driver */
static int find_alloc(uintptr_t p, size_t n);
CUresult cuPointerGetAttribute(void* out, CUpointer_attribute attr, CUdeviceptr p) {
    int id = find_alloc((uintptr_t)p, 1);
    if (id < 0) return CUDA_ERROR_INVALID_VALUE;
    if (attr == CU_POINTER_ATTRIBUTE_MEMORY_TYPE) { *(unsigned int*)out = allocs[id].host ? CU_MEMORYTYPE_HOST : CU_MEMORYTYPE_DEVICE; return CUDA_SUCCESS; }
    if (attr == CU_POINTER_ATTRIBUTE_DEVICE_POINTER) { *(CUdeviceptr*)out = p; return CUDA_SUCCESS; }
    return CUDA_ERROR_INVALID_VALUE;
}
CUresult cuDevicePrimaryCtxRetain(CUcontext* c, CUdevice d) { (void)d; *c = (CUcontext)&fake_ctx; return CUDA_SUCCESS; }
CUresult cuDevicePrimaryCtxRelease_v2(CUdevice d) { (void)d; return CUDA_SUCCESS; }
static CUcontext cur_ctx;
CUresult cuCtxSetCurrent(CUcontext c) { cur_ctx = c; return CUDA_SUCCESS; }
CUresult cuCtxGetCurrent(CUcontext* c) { *c = cur_ctx; return CUDA_SUCCESS; }
static const unsigned char* module_image;
CUresult cuModuleLoadData(CUmodule* m, const void* image) {
    if (memcmp(image, "\x7f" "ELF", 4)) return bad("module image is not an ELF cubin");
    module_image = image;
    *m = (CUmodule)&fake_mod; return CUDA_SUCCESS;
}
CUresult cuModuleUnload(CUmodule m) { (void)m; return CUDA_SUCCESS; }
/* as the driver: a name is found only if it is a function symbol of the loaded cubin's .symtab */
static int image_has_function(const char* name) {
    const Elf64_Ehdr* eh = (const Elf64_Ehdr*)module_image;
    const Elf64_Shdr* sh = (const Elf64_Shdr*)(module_image + eh->e_shoff);
    for (int i = 0; i < eh->e_shnum; ++i) {
        if (sh[i].sh_type != SHT_SYMTAB) continue;
        const Elf64_Sym* sym = (const Elf64_Sym*)(module_image + sh[i].sh_offset);
        const char* str = (const char*)module_image + sh[sh[i].sh_link].sh_offset;
        for (size_t k = 0; k < sh[i].sh_size / sizeof *sym; ++k)
            if (ELF64_ST_TYPE(sym[k].st_info) == STT_FUNC && !strcmp(str + sym[k].st_name, name)) return 1;
    }
    return 0;
}
CUresult cuModuleGetFunction(CUfunction* f, CUmodule m, const char* name) {
    (void)m;
    for (int i = 0; i < n_fns; ++i) if (!strcmp(fns[i].name, name)) { *f = (CUfunction)&fns[i]; return CUDA_SUCCESS; }
    if (!module_image || !image_has_function(name)) {
        LOG("{\"op\":\"error\",\"what\":\"no function %s in the module\"}", name);
        return CUDA_ERROR_NOT_FOUND;
    }
    if (n_fns >= 512) return CUDA_ERROR_INVALID_VALUE;
    snprintf(fns[n_fns].name, sizeof fns[0].name, "%s", name); fns[n_fns].max_dyn_smem = 48 * 1024;
    *f = (CUfunction)&fns[n_fns++];
    return CUDA_SUCCESS;
}
CUresult cuFuncSetAttribute(CUfunction f, CUfunction_attribute a, int v) {
    if (a == CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES) {
        if (v > 232448) return bad("dynamic shared memory above the 227 KiB opt-in limit");
        ((mock_fn*)f)->max_dyn_smem = v;
    }
    return CUDA_SUCCESS;
}
CUresult cuOccupancyMaxActiveBlocksPerMultiprocessor(int* n, CUfunction f, int block, size_t smem) {
    (void)f;
    int by_threads = 2048 / (block > 0 ? block : 1), by_smem = smem ? (int)((228u * 1024u) / (smem + 1024u)) : 32;
    int v = by_threads < by_smem ? by_threads : by_smem;
    *n = v > 32 ? 32 : v;
    return CUDA_SUCCESS;
}
static int stream_id(CUstream s) { return s ? (int)((uintptr_t)s & 0xFFFF) : 0; }
CUresult cuLaunchKernel(CUfunction f, unsigned gx, unsigned gy, unsigned gz, unsigned bx, unsigned by, unsigned bz,
                        unsigned smem, CUstream s, void** params, void** extra) {
    (void)extra;
    mock_fn* fn = (mock_fn*)f;
    if (!gx || !gy || !gz || !bx || bx * by * bz > 1024) return bad("launch geometry");
    if ((int)smem > fn->max_dyn_smem) return bad("dynamic shared memory above the function's limit");
    log_open();
    if (logf) {
        fprintf(logf, "{\"op\":\"launch\",\"name\":\"%s\",\"grid\":%u,\"block\":%u,\"smem\":%u,\"stream\":%d,\"arg0\":\"", fn->name,
                gx * gy * gz, bx * by * bz, smem, stream_id(s));
        /* xmr_* kernels take the 128-byte argument block first; the helper kernels take small scalars (dump 8 bytes) */
        const int is_args = strncmp(fn->name, "xmr_", 4) == 0 && strstr(fn->name, "_nc") != NULL;
        const unsigned char* p = (const unsigned char*)params[0];
        for (int i = 0; i < (is_args ? 128 : 8); ++i) fprintf(logf, "%02x", p[i]);
        fprintf(logf, "\"}\n"); fflush(logf);
    }
    const char* tally = getenv("MOCK_CUDA_TALLY");                        /* "errors,dwc,syncs,injected,first": what a kernel would have counted */
    if (tally && strncmp(fn->name, "xmr_", 4) == 0 && strstr(fn->name, "_nc")) {
        unsigned long long v[5] = { 0, 0, 0, 0, ~0ull };
        sscanf(tally, "%llu,%llu,%llu,%llu,%llu", &v[0], &v[1], &v[2], &v[3], &v[4]);
        unsigned long long* c = *(unsigned long long**)((const unsigned char*)params[0] + 40);   /* xmr_args.counters */
        if (find_alloc((uintptr_t)c, 5 * 8) < 0) return bad("counters pointer in the argument block");
        for (int i = 0; i < 4; ++i) c[i] += v[i];
        if (v[4] < c[4]) c[4] = v[4];
    }
    if (!strcmp(fn->name, "xmr_counters_reset")) {                         /* the one kernel whose effect the host relies on */
        unsigned long long* c = *(unsigned long long**)params[0];
        if (find_alloc((uintptr_t)c, 5 * 8) < 0) return bad("counters pointer");
        c[0] = c[1] = c[2] = c[3] = 0; c[4] = ~0ull;
    }
    return CUDA_SUCCESS;
}
CUresult cuMemAlloc_v2(CUdeviceptr* p, size_t n) { return do_alloc(p, n, 0); }
CUresult cuMemFree_v2(CUdeviceptr p) { return do_free(p); }
CUresult cuMemPoolCreate(CUmemoryPool* pool, const CUmemPoolProps* props) {
    if (props->allocType != CU_MEM_ALLOCATION_TYPE_PINNED || props->location.type != CU_MEM_LOCATION_TYPE_DEVICE) return bad("pool props");
    *pool = (CUmemoryPool)&fake_mod; return CUDA_SUCCESS;
}
CUresult cuMemPoolDestroy(CUmemoryPool p) { (void)p; return CUDA_SUCCESS; }
CUresult cuMemPoolSetAttribute(CUmemoryPool p, CUmemPool_attribute a, void* v) { (void)p; (void)a; (void)v; return CUDA_SUCCESS; }
CUresult cuMemAllocFromPoolAsync(CUdeviceptr* p, size_t n, CUmemoryPool pool, CUstream s) { (void)pool; (void)s; return do_alloc(p, n, 0); }
CUresult cuMemFreeAsync(CUdeviceptr p, CUstream s) { (void)s; return do_free(p); }
static CUresult copy(const char* op, void* dst, const void* src, size_t n, uintptr_t dev, CUstream s) {
    int id = find_alloc(dev, n);
    if (id < 0) return bad("copy outside a live device allocation");
    memcpy(dst, src, n);
    LOG("{\"op\":\"%s\",\"alloc\":%d,\"offset\":%zu,\"bytes\":%zu,\"host\":%llu,\"stream\":%d}", op, id, (size_t)(dev - allocs[id].base), n,
        (unsigned long long)(uintptr_t)(op[0] == 'h' ? src : dst), stream_id(s));
    return CUDA_SUCCESS;
}
CUresult cuMemcpyHtoDAsync_v2(CUdeviceptr d, const void* h, size_t n, CUstream s) { return copy("h2d", (void*)(uintptr_t)d, h, n, (uintptr_t)d, s); }
CUresult cuMemcpyDtoHAsync_v2(void* h, CUdeviceptr d, size_t n, CUstream s) { return copy("d2h", h, (const void*)(uintptr_t)d, n, (uintptr_t)d, s); }
CUresult cuMemcpyDtoDAsync_v2(CUdeviceptr dst, CUdeviceptr src, size_t n, CUstream s) {
    (void)s;
    if (find_alloc((uintptr_t)dst, n) < 0 || find_alloc((uintptr_t)src, n) < 0) return bad("d2d outside a live allocation");
    memmove((void*)(uintptr_t)dst, (const void*)(uintptr_t)src, n);
    return CUDA_SUCCESS;
}
CUresult cuMemsetD8Async(CUdeviceptr d, unsigned char v, size_t n, CUstream s) {
    (void)s;
    if (find_alloc((uintptr_t)d, n) < 0) return bad("memset outside a live allocation");
    memset((void*)(uintptr_t)d, v, n); return CUDA_SUCCESS;
}
CUresult cuMemHostAlloc(void** p, size_t n, unsigned int flags) { (void)flags; CUdeviceptr d; CUresult r = do_alloc(&d, n, 1); *p = (void*)(uintptr_t)d; return r; }
CUresult cuMemFreeHost(void* p) { return do_free((CUdeviceptr)(uintptr_t)p); }
CUresult cuStreamCreate(CUstream* s, unsigned int flags) { (void)flags; *s = (CUstream)(uintptr_t)(0x1000 + ++n_streams); return CUDA_SUCCESS; }
CUresult cuStreamDestroy_v2(CUstream s) { (void)s; return CUDA_SUCCESS; }
CUresult cuStreamSynchronize(CUstream s) { LOG("{\"op\":\"stream_sync\",\"stream\":%d}", stream_id(s)); return CUDA_SUCCESS; }
CUresult cuEventCreate(CUevent* e, unsigned int flags) { (void)flags; *e = (CUevent)&fake_mod; return CUDA_SUCCESS; }
CUresult cuEventRecord(CUevent e, CUstream s) { (void)e; LOG("{\"op\":\"event_record\",\"stream\":%d}", stream_id(s)); return CUDA_SUCCESS; }
CUresult cuEventDestroy_v2(CUevent e) { (void)e; return CUDA_SUCCESS; }
CUresult cuStreamWaitEvent(CUstream s, CUevent e, unsigned int f) { (void)e; (void)f; LOG("{\"op\":\"wait_event\",\"stream\":%d}", stream_id(s)); return CUDA_SUCCESS; }
CUresult cuGetErrorString(CUresult r, const char** s) { (void)r; *s = "mock driver error"; return CUDA_SUCCESS; }
/* IPC: the "handle" is the pointer itself; MOCK_IPC_FAIL=1 makes the open fail (no peer access) */
CUresult cuIpcGetMemHandle(CUipcMemHandle* h, CUdeviceptr p) { memset(h, 0, sizeof *h); memcpy(h, &p, sizeof p); LOG("{\"op\":\"ipc_get\",\"ptr\":%llu}", (unsigned long long)p); return CUDA_SUCCESS; }
CUresult cuIpcOpenMemHandle_v2(CUdeviceptr* p, CUipcMemHandle h, unsigned int flags) {
    if (getenv("MOCK_IPC_FAIL")) return CUDA_ERROR_PEER_ACCESS_UNSUPPORTED;
    memcpy(p, &h, sizeof *p); LOG("{\"op\":\"ipc_open\",\"ptr\":%llu,\"flags\":%u}", (unsigned long long)*p, flags); return CUDA_SUCCESS;
}
CUresult cuIpcCloseMemHandle(CUdeviceptr p) { LOG("{\"op\":\"ipc_close\",\"ptr\":%llu}", (unsigned long long)p); return CUDA_SUCCESS; }

CUresult cuTensorMapEncodeTiled(CUtensorMap* map, CUtensorMapDataType dt, cuuint32_t rank, void* addr, const cuuint64_t* gdim,
                                const cuuint64_t* gstr, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapInterleave il,
                                CUtensorMapSwizzle swz, CUtensorMapL2promotion l2, CUtensorMapFloatOOBfill oob) {
    (void)l2; (void)oob;
    size_t es;
    switch (dt) {
    case CU_TENSOR_MAP_DATA_TYPE_UINT8: es = 1; break;
    case CU_TENSOR_MAP_DATA_TYPE_BFLOAT16: es = 2; break;
    case CU_TENSOR_MAP_DATA_TYPE_UINT32: case CU_TENSOR_MAP_DATA_TYPE_FLOAT32: es = 4; break;
    default: return bad("tensor map data type");
    }
    if (rank < 1 || rank > 5) return bad("tensor map rank");
    if (((uintptr_t)addr) & 15u) return bad("tensor map: global address must be 16-byte aligned");
    if (il != CU_TENSOR_MAP_INTERLEAVE_NONE) return bad("tensor map interleave");
    size_t extent = es;
    for (cuuint32_t i = 0; i < rank; ++i) {
        if (gdim[i] < 1 || gdim[i] > (1ull << 32)) return bad("tensor map: globalDim out of range");
        if (box[i] < 1 || box[i] > 256) return bad("tensor map: boxDim must be 1..256");
        if (estr[i] < 1 || estr[i] > 8) return bad("tensor map: elementStrides");
        if (i > 0) {
            if (gstr[i - 1] % 16 || gstr[i - 1] >= (1ull << 40)) return bad("tensor map: globalStrides must be multiples of 16 below 2^40");
            extent += (size_t)(gdim[i] - 1) * gstr[i - 1];
        } else extent += (size_t)(gdim[0] - 1) * es;
    }
    const size_t inner = (size_t)box[0] * es;
    if (inner % 16) return bad("tensor map: inner box extent must be a multiple of 16 bytes");
    const size_t lim = swz == CU_TENSOR_MAP_SWIZZLE_32B ? 32 : swz == CU_TENSOR_MAP_SWIZZLE_64B ? 64 : swz == CU_TENSOR_MAP_SWIZZLE_NONE ? 256 * es : 128;
    if (inner > lim) return bad("tensor map: inner box extent exceeds the swizzle span");
    if (find_alloc((uintptr_t)addr, extent) < 0) return bad("tensor map covers memory outside a live allocation");
    size_t box_bytes = es; for (cuuint32_t i = 0; i < rank; ++i) box_bytes *= box[i];
    memset(map, 0, sizeof *map);
    LOG("{\"op\":\"tmap\",\"addr\":%llu,\"rank\":%u,\"elem\":%zu,\"dim0\":%llu,\"dim1\":%llu,\"box0\":%u,\"box1\":%u,\"box_bytes\":%zu,\"swizzle\":%d}",
        (unsigned long long)(uintptr_t)addr, rank, es, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 1), box[0], rank > 1 ? box[1] : 1, box_bytes, (int)swz);
    return CUDA_SUCCESS;
}
