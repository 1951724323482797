// host.cpp — the headless launch surface behind include/simlod_b200.h.
//
// Restates, on the CUDA driver API like the reference, the host side of the hot path:
//   initCuda / initCudaProgram   main_progressive_octree.cpp:272-281, 549-642
//   getUniforms                  :283-331        resetCUDA     :333-361
//   updateOctree                 :364-428        renderCUDA    :465-546
//   uploader step                :1033-1056      stats readback :1201-1216
// The three programs are sm_90a cubins embedded in this library (the reference NVRTC-compiles
// its sources at start-up, CudaModularProgram.h:62-135); simlod_use_module swaps one of them
// for an external cubin with the same kernel name (the reference's hot reload, :181-184).
// There is no CPU fallback: without a device or a loadable cubin every call fails.
#include "../../include/simlod_b200.h"
#include <cuda.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <sched.h>
#if defined(__x86_64__)
#include <emmintrin.h>
#endif
#include <unistd.h>
#include <sys/syscall.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <cstdarg>
#include <cstdio>
#include <cctype>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

extern "C" {
extern const unsigned char simlod_cubin_construct[];
extern const unsigned char simlod_cubin_render[];
extern const unsigned char simlod_cubin_reset[];
extern const unsigned char simlod_cubin_util[];
extern const unsigned char simlod_cubin_partition[];
extern const unsigned char simlod_cubin_las[];
extern const unsigned char simlod_cubin_gen[];
}

namespace {

thread_local std::string g_error;

int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_error = buf;
    return code;
}


// ------------------------------------------------------------------------------------------
// The driver API is bound at run time (dlopen libcuda.so.1) so that the library can be loaded
// and its exports inspected on a machine without a GPU driver; every entry point that touches
// the device fails with SIMLOD_ERR_CUDA there. There is no other code path.
// ------------------------------------------------------------------------------------------
#define DRV_LIST(X) X(cuArray3DCreate) X(cuArrayDestroy) X(cuCtxSetCurrent) X(cuCtxSynchronize) X(cuDeviceGet) X(cuDeviceGetAttribute) X(cuDeviceGetPCIBusId) X(cuDevicePrimaryCtxRelease) X(cuDevicePrimaryCtxRetain) X(cuEventCreate) X(cuEventDestroy) X(cuEventElapsedTime) X(cuEventQuery) X(cuEventRecord) X(cuEventSynchronize) X(cuGetErrorString) X(cuInit) X(cuLaunchCooperativeKernel) X(cuLaunchKernel) X(cuMemAlloc) X(cuMemFree) X(cuMemFreeHost) X(cuMemGetInfo) X(cuMemHostAlloc) X(cuMemcpy2D) X(cuMemcpyDtoDAsync) X(cuMemcpyDtoH) X(cuMemcpyDtoHAsync) X(cuMemcpyHtoD) X(cuMemcpyHtoDAsync) X(cuMemsetD32Async) X(cuMemsetD8) X(cuMemsetD8Async) X(cuModuleGetFunction) X(cuModuleLoadData) X(cuModuleUnload) X(cuOccupancyMaxActiveBlocksPerMultiprocessor) X(cuStreamCreate) X(cuStreamDestroy) X(cuStreamSynchronize) X(cuStreamWaitEvent) X(cuSurfObjectCreate) X(cuSurfObjectDestroy)
#define DRV_STR2(x) #x
#define DRV_STR(x) DRV_STR2(x)
struct DriverApi {
#define X(name) decltype(&name) p_##name = nullptr;
    DRV_LIST(X)
#undef X
    void* handle = nullptr;
    bool loaded = false;
};
DriverApi drv;
#define D(name) drv.p_##name

int loadDriver() {
    if (drv.loaded) return SIMLOD_OK;
    drv.handle = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!drv.handle) return fail(SIMLOD_ERR_CUDA, "cannot load libcuda.so.1 (%s): a CUDA driver and an H100 are required, there is no CPU path", dlerror());
#define X(name) drv.p_##name = reinterpret_cast<decltype(&name)>(dlsym(drv.handle, DRV_STR(name))); \
    if (!drv.p_##name) return fail(SIMLOD_ERR_CUDA, "libcuda.so.1 lacks %s", DRV_STR(name));
    DRV_LIST(X)
#undef X
    drv.loaded = true;
    return SIMLOD_OK;
}

#define CU(call)                                                                              \
    do {                                                                                      \
        CUresult _r = (call);                                                                 \
        if (_r != CUDA_SUCCESS) {                                                             \
            const char* _s = nullptr; D(cuGetErrorString)(_r, &_s);                              \
            return fail(SIMLOD_ERR_CUDA, "%s failed: %s (%d) at %s:%d", #call, _s ? _s : "?", (int)_r, __FILE__, __LINE__); \
        }                                                                                     \
    } while (0)

constexpr uint64_t RING_SLOTS = SIMLOD_BATCH_STREAM_SIZE;
constexpr uint64_t SLOT_POINTS = SIMLOD_MAX_BATCH_SIZE;
constexpr uint64_t FB_OFFSET = 31200144;       // render.cu:1108-1123 carve-out
constexpr uint64_t L2_FLUSH_BYTES = 512ull << 20;

struct Program {
    CUmodule module = nullptr;
    CUfunction fn = nullptr;
    bool builtin = true;
};

}  // namespace

#include "loader_pool.h"

struct SimlodContext {
    CUdevice device = 0;
    CUcontext primary = nullptr;
    int numSMs = 0;
    CUstream streamMain = nullptr, streamUpload = nullptr;
    CUevent evStart = nullptr, evEnd = nullptr, evTotalStart = nullptr, evTotalEnd = nullptr;
    CUevent evBurst[8][2] = {};        // event pairs for launches enqueued back to back
    CUevent evSlot[RING_SLOTS] = {};    // recorded on the upload stream when the batch in that ring slot has been published
    SimlodConfig cfg{};
    SimlodUniforms uniforms{};
    SimlodBuffers buf{};
    CUdeviceptr numBatchesUploaded = 0, batchSizes = 0, frameStart = 0, cudaprint = 0, scratch4 = 0, flushBuf = 0;
    CUarray colorArray = nullptr;
    CUsurfObject surface = 0;
    SimlodStats* hStats = nullptr;     // pinned
    SimlodStats* hStatsRing = nullptr; // pinned, one snapshot per launch in flight (8)
    struct PublishMirror { uint32_t sizes[RING_SLOTS]; uint32_t count; uint32_t pad[13]; };   // 256 B
    PublishMirror* hPublish = nullptr; // pinned, 16 snapshots of {batchSizes[50], numBatchesUploaded} for grouped publication
    CUevent evPublish[16] = {};        // the copies out of mirror i have completed
    uint32_t hostSizes[RING_SLOTS] = {};   // what batchSizes[] holds on the device once everything enqueued has run
    uint32_t unpublished = 0;          // batches copied into the ring but not yet published (sizes + counter)
    uint32_t publishIndex = 0;
    CUevent evStatsDone[8] = {};       // the snapshot behind launch slot k has landed
    Program programs[3];
    CUmodule utilModule = nullptr, lasModule = nullptr, partitionModule = nullptr, genModule = nullptr;
    CUfunction fnGenUniform = nullptr, fnGenTerrain = nullptr, fnGenShell = nullptr;
    CUfunction fnPartCount = nullptr, fnPartScan = nullptr, fnPartScatter = nullptr;
    CUfunction fnPartWait = nullptr, fnComposite = nullptr, fnPeerSignal = nullptr;
    CUdeviceptr partScratch = 0;       // spatial exchange: PART_SLOTS x (blockHist | blockBase | totals | cellCounts), then blocksDone, timedOut
    struct PartSlot { uint64_t points = 0; uint32_t count = 0; bool valid = false; } partSlots[64];   // counted batches awaiting their scatter
    uint32_t partNextSlot = 0;
    CUfunction fnLas = nullptr;
    CUdeviceptr lasStaging = 0;        // raw LAS records of the batch being decoded
    void* pinnedPool = nullptr;        // POOL_SLOTS x 16 MB page-locked staging slots of the file streamer
    LoaderPool* loaderPool = nullptr;
    CUevent evPool[32] = {};           // H2D copy out of pool slot i has been enqueued and completed
    CUfunction fnRcp = nullptr, fnFill = nullptr;
    uint32_t uploaded = 0;             // batches published to the device
    uint32_t processed = 0;            // Stats::batchletIndex as last read
    uint64_t launches = 0;
    uint32_t constructBlocks = 0, renderBlocks = 0;
    int numaNode = -1;                 // host NUMA node the page-locked buffers were placed on (-1: unknown)
    uint64_t frameCounter = 0;
};

namespace {

int devAlloc(uint64_t* out, uint64_t bytes) {
    CUdeviceptr p = 0;
    CU(D(cuMemAlloc)(&p, (size_t)bytes));
    *out = (uint64_t)p;
    return SIMLOD_OK;
}
#define ALLOC(field, bytes) do { int _rc = devAlloc(&(field), (bytes)); if (_rc) return _rc; } while (0)

// Page-locked host memory should live on the NUMA node the GPU hangs off: the copy engine then reads local DRAM
// instead of crossing the socket interconnect (which all ranks of a multi-GPU job would share). The driver
// allocates on the node of the calling thread, so the thread is parked on that node's CPUs for the call.
struct NumaLocal {
    cpu_set_t old;
    bool active = false, policy = false;
    int node = -1;
    explicit NumaLocal(SimlodContext* ctx) {
        // the host NUMA node closest to the device: the driver's own answer first, sysfs second
        int attr = -1;
        if (D(cuDeviceGetAttribute)(&attr, (CUdevice_attribute)134 /* CU_DEVICE_ATTRIBUTE_HOST_NUMA_ID */, ctx->device) == CUDA_SUCCESS && attr >= 0) node = attr;
        if (node < 0) {
            char bus[32] = {0};
            if (D(cuDeviceGetPCIBusId)(bus, (int)sizeof(bus), ctx->device) != CUDA_SUCCESS) return;
            for (char* c = bus; *c; c++) *c = (char)tolower(*c);
            char path[128];
            snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
            if (FILE* f = fopen(path, "r")) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
        }
        if (node < 0) return;
        ctx->numaNode = node;
        // page placement follows the allocating thread: prefer the node for its allocations (works where the container lets
        // set_mempolicy through) and park the thread on the node's CPUs (first touch) for the duration of the call
        unsigned long mask[16] = {0};
        if (node < (int)(sizeof(mask) * 8)) {
            mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
            policy = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof(mask) * 8) == 0;
        }
        char path[128];
        snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
        char list[4096] = {0};
        if (FILE* f = fopen(path, "r")) { if (!fgets(list, sizeof(list), f)) list[0] = 0; fclose(f); }
        cpu_set_t want;
        CPU_ZERO(&want);
        for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
            int a = 0, b = 0;
            int n = sscanf(tok, "%d-%d", &a, &b);
            if (n == 1) b = a;
            if (n >= 1) for (int c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET(c, &want);
        }
        if (sched_getaffinity(0, sizeof(old), &old) != 0) return;
        CPU_AND(&want, &want, &old);
        if (CPU_COUNT(&want) == 0) return;
        active = sched_setaffinity(0, sizeof(want), &want) == 0;
    }
    ~NumaLocal() {
        if (active) sched_setaffinity(0, sizeof(old), &old);
        if (policy) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
    }
};

const char* kernelName(int program) {
    switch (program) {
        case SIMLOD_PROGRAM_CONSTRUCT: return "kernel_construct";
        case SIMLOD_PROGRAM_RENDER: return "kernel_render";
        case SIMLOD_PROGRAM_RESET: return "kernel";
    }
    return nullptr;
}
const unsigned char* builtinImage(int program) {
    switch (program) {
        case SIMLOD_PROGRAM_CONSTRUCT: return simlod_cubin_construct;
        case SIMLOD_PROGRAM_RENDER: return simlod_cubin_render;
        case SIMLOD_PROGRAM_RESET: return simlod_cubin_reset;
    }
    return nullptr;
}

int setCurrent(SimlodContext* ctx) {
    if (!ctx) return fail(SIMLOD_ERR_INVALID, "null context");
    CU(D(cuCtxSetCurrent)(ctx->primary));
    return SIMLOD_OK;
}

int computeGrids(SimlodContext* ctx) {
    // updateOctree: numGroups = numSMs (main.cpp:370-371); renderCUDA: occupancy * numSMs (main.cpp:493-497).
    // Our construct kernel is written for any cooperative grid, so by default both use the occupancy query.
    int occ = 0;
    CU(D(cuOccupancyMaxActiveBlocksPerMultiprocessor)(&occ, ctx->programs[SIMLOD_PROGRAM_CONSTRUCT].fn, 256, 0));
    int per = ctx->cfg.construct_blocks_per_sm > 0 ? std::min(ctx->cfg.construct_blocks_per_sm, occ) : occ;
    if (per < 1) return fail(SIMLOD_ERR_MODULE, "kernel_construct cannot be resident with 256 threads");
    ctx->constructBlocks = (uint32_t)(per * ctx->numSMs);
    CU(D(cuOccupancyMaxActiveBlocksPerMultiprocessor)(&occ, ctx->programs[SIMLOD_PROGRAM_RENDER].fn, 256, 0));
    per = ctx->cfg.render_blocks_per_sm > 0 ? std::min(ctx->cfg.render_blocks_per_sm, occ) : occ;
    if (per < 1) return fail(SIMLOD_ERR_MODULE, "kernel_render cannot be resident with 256 threads");
    ctx->renderBlocks = (uint32_t)(per * ctx->numSMs);
    return SIMLOD_OK;
}

int loadProgram(SimlodContext* ctx, int program, const void* image, bool builtin) {
    CUmodule mod = nullptr;
    CUresult r = D(cuModuleLoadData)(&mod, image);
    if (r != CUDA_SUCCESS) {
        const char* s = nullptr; D(cuGetErrorString)(r, &s);
        return fail(SIMLOD_ERR_MODULE, "D(cuModuleLoadData)(%s) failed: %s", kernelName(program), s ? s : "?");
    }
    CUfunction fn = nullptr;
    r = D(cuModuleGetFunction)(&fn, mod, kernelName(program));
    if (r != CUDA_SUCCESS) { D(cuModuleUnload)(mod); return fail(SIMLOD_ERR_MODULE, "module does not export %s", kernelName(program)); }
    Program& p = ctx->programs[program];
    if (p.module) D(cuModuleUnload)(p.module);
    p.module = mod; p.fn = fn; p.builtin = builtin;
    return SIMLOD_OK;
}

int readStats(SimlodContext* ctx) {
    CU(D(cuMemcpyDtoHAsync)(ctx->hStats, ctx->buf.stats, sizeof(SimlodStats), ctx->streamMain));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    ctx->processed = ctx->hStats->batchletIndex;
    return SIMLOD_OK;
}

// Stats::dbg carries kernel_construct's sticky capacity flags (construct.cu: ERR_*); bit 7 (a point far outside the
// box) is informational
int checkOverflow(SimlodContext* ctx) {
    // bits 0, 3, 5 (spill buffer, nodes[], split list full) only POSTPONE a split — no sample is lost, the octree stays valid,
    // the bit stays visible in Stats::dbg; bits 1, 2, 4, 6 mean voxels or points were dropped: that is an error
    const uint32_t flags = ctx->hStats->dbg & (uint32_t)SIMLOD_DBG_FATAL_MASK;
    if (flags) return fail(SIMLOD_ERR_OVERFLOW, "kernel_construct dropped samples: a per-batch capacity was exceeded (Stats::dbg = 0x%x: 2 voxel backlog, 4 chunk directory, 16 chunk stack, 64 leaf rows, 256 internal); reset to clear", ctx->hStats->dbg);
    return SIMLOD_OK;
}

// Publication of a GROUP of batches whose points have been copied into their ring slots (uploadCommon with publish =
// false): ONE copy of the 50 slot sizes and ONE of the counter, out of a pinned snapshot, instead of two small
// operations per batch. With a device-resident source the 40 memsets behind 20 batch copies were what the next launch
// waited for: 0.3 ms of idle GPU between launches (tools/launch_gaps.py), 10 % of the whole insertion.
int publishPending(SimlodContext* ctx) {
    if (ctx->unpublished == 0) return SIMLOD_OK;
    const uint32_t m = ctx->publishIndex++ % 16u;
    if (ctx->publishIndex > 16u) CU(D(cuEventSynchronize)(ctx->evPublish[m]));       // the snapshot's previous copies have left it
    SimlodContext::PublishMirror* pm = &ctx->hPublish[m];
    memcpy(pm->sizes, ctx->hostSizes, sizeof(pm->sizes));
    pm->count = ctx->uploaded;
    CU(D(cuMemcpyHtoDAsync)(ctx->batchSizes, pm->sizes, sizeof(pm->sizes), ctx->streamUpload));        // main.cpp:1047-1050: sizes first,
    CU(D(cuMemcpyHtoDAsync)(ctx->numBatchesUploaded, &pm->count, 4, ctx->streamUpload));                // then the global counter
    CU(D(cuEventRecord)(ctx->evPublish[m], ctx->streamUpload));
    for (uint32_t k = ctx->unpublished; k > 0; k--) CU(D(cuEventRecord)(ctx->evSlot[(ctx->uploaded - k) % RING_SLOTS], ctx->streamUpload));
    ctx->unpublished = 0;
    return SIMLOD_OK;
}

int publishBatch(SimlodContext* ctx, uint32_t slot, uint32_t count) {
    // main.cpp:1047-1050: the size of the slot first, then the global counter, in stream order after the copy
    int prc = publishPending(ctx); if (prc) return prc;
    ctx->hostSizes[slot] = count;
    CU(D(cuMemsetD32Async)(ctx->batchSizes + 4ull * slot, count, 1, ctx->streamUpload));
    ctx->uploaded++;
    CU(D(cuMemsetD32Async)(ctx->numBatchesUploaded, ctx->uploaded, 1, ctx->streamUpload));
    CU(D(cuEventRecord)(ctx->evSlot[slot], ctx->streamUpload));
    return SIMLOD_OK;
}

// enqueue one kernel_construct launch between the event pair `slot` without waiting for it
int enqueueConstruct(SimlodContext* ctx, int slot, CUdeviceptr pointsBase = 0) {
    SimlodUniforms u = ctx->uniforms;
    u.frameCounter = ctx->frameCounter;
    CUdeviceptr ring = pointsBase ? pointsBase : ctx->buf.ring, momentary = ctx->buf.momentary, persistent = ctx->buf.persistent, nodes = ctx->buf.nodes,
                stats = ctx->buf.stats, frameStart = ctx->frameStart, cudaprint = ctx->cudaprint,
                nbu = ctx->numBatchesUploaded, bs = ctx->batchSizes;
    void* args[] = {&u, &ring, &momentary, &persistent, &nodes, &stats, &frameStart, &cudaprint, &nbu, &bs};   // main.cpp:374-382
    CU(D(cuEventRecord)(ctx->evBurst[slot][0], ctx->streamMain));
    CU(D(cuLaunchCooperativeKernel)(ctx->programs[SIMLOD_PROGRAM_CONSTRUCT].fn, ctx->constructBlocks, 1, 1, 256, 1, 1, 0, ctx->streamMain, args));
    CU(D(cuEventRecord)(ctx->evBurst[slot][1], ctx->streamMain));
    ctx->launches++;
    return SIMLOD_OK;
}

int launchConstruct(SimlodContext* ctx, float* ms) {
    SimlodUniforms u = ctx->uniforms;
    u.frameCounter = ctx->frameCounter;
    CUdeviceptr ring = ctx->buf.ring, momentary = ctx->buf.momentary, persistent = ctx->buf.persistent, nodes = ctx->buf.nodes,
                stats = ctx->buf.stats, frameStart = ctx->frameStart, cudaprint = ctx->cudaprint,
                nbu = ctx->numBatchesUploaded, bs = ctx->batchSizes;
    void* args[] = {&u, &ring, &momentary, &persistent, &nodes, &stats, &frameStart, &cudaprint, &nbu, &bs};   // main.cpp:374-382
    CU(D(cuEventRecord)(ctx->evStart, ctx->streamMain));
    CU(D(cuLaunchCooperativeKernel)(ctx->programs[SIMLOD_PROGRAM_CONSTRUCT].fn, ctx->constructBlocks, 1, 1, 256, 1, 1, 0, ctx->streamMain, args));
    CU(D(cuEventRecord)(ctx->evEnd, ctx->streamMain));
    ctx->launches++;
    CU(D(cuEventSynchronize)(ctx->evEnd));
    if (ms) CU(D(cuEventElapsedTime)(ms, ctx->evStart, ctx->evEnd));
    return SIMLOD_OK;
}

}  // namespace

extern "C" {

const char* simlod_last_error(void) { return g_error.c_str(); }

// everything simlod_create sets up after the primary context is retained; on failure the caller destroys the
// partially built context (simlod_destroy releases whatever exists)
static int createResources(SimlodContext* ctx, const SimlodConfig* config) {
    CU(D(cuCtxSetCurrent)(ctx->primary));
    CU(D(cuDeviceGetAttribute)(&ctx->numSMs, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, ctx->device));
    int coop = 0;
    CU(D(cuDeviceGetAttribute)(&coop, CU_DEVICE_ATTRIBUTE_COOPERATIVE_LAUNCH, ctx->device));
    if (!coop) return fail(SIMLOD_ERR_CUDA, "device does not support cooperative launches");
    CU(D(cuStreamCreate)(&ctx->streamMain, CU_STREAM_NON_BLOCKING));
    CU(D(cuStreamCreate)(&ctx->streamUpload, CU_STREAM_NON_BLOCKING));      // main.cpp:276
    CU(D(cuEventCreate)(&ctx->evStart, CU_EVENT_DEFAULT));
    CU(D(cuEventCreate)(&ctx->evEnd, CU_EVENT_DEFAULT));
    CU(D(cuEventCreate)(&ctx->evTotalStart, CU_EVENT_DEFAULT));
    CU(D(cuEventCreate)(&ctx->evTotalEnd, CU_EVENT_DEFAULT));
    for (int i = 0; i < 8; i++) for (int j = 0; j < 2; j++) CU(D(cuEventCreate)(&ctx->evBurst[i][j], CU_EVENT_DEFAULT));
    for (uint64_t i = 0; i < RING_SLOTS; i++) CU(D(cuEventCreate)(&ctx->evSlot[i], CU_EVENT_DISABLE_TIMING));

    // programs (main.cpp:603-626)
    for (int p = 0; p < 3; p++) {
        int rc = loadProgram(ctx, p, builtinImage(p), true);
        if (rc != SIMLOD_OK) return rc;
    }
    CU(D(cuModuleLoadData)(&ctx->utilModule, simlod_cubin_util));
    CU(D(cuModuleGetFunction)(&ctx->fnRcp, ctx->utilModule, "simlod_util_rcp"));
    CU(D(cuModuleGetFunction)(&ctx->fnFill, ctx->utilModule, "simlod_util_fill"));
    CU(D(cuModuleLoadData)(&ctx->lasModule, simlod_cubin_las));
    CU(D(cuModuleGetFunction)(&ctx->fnLas, ctx->lasModule, "simlod_las_decode"));
    CU(D(cuModuleLoadData)(&ctx->genModule, simlod_cubin_gen));
    CU(D(cuModuleGetFunction)(&ctx->fnGenUniform, ctx->genModule, "simlod_gen_uniform"));
    CU(D(cuModuleGetFunction)(&ctx->fnGenTerrain, ctx->genModule, "simlod_gen_terrain"));
    CU(D(cuModuleGetFunction)(&ctx->fnGenShell, ctx->genModule, "simlod_gen_shell"));
    CU(D(cuModuleLoadData)(&ctx->partitionModule, simlod_cubin_partition));
    CU(D(cuModuleGetFunction)(&ctx->fnPartCount, ctx->partitionModule, "simlod_partition_count"));
    CU(D(cuModuleGetFunction)(&ctx->fnPartScan, ctx->partitionModule, "simlod_partition_scan"));
    CU(D(cuModuleGetFunction)(&ctx->fnPartScatter, ctx->partitionModule, "simlod_partition_scatter"));
    CU(D(cuModuleGetFunction)(&ctx->fnPartWait, ctx->partitionModule, "simlod_partition_wait"));
    CU(D(cuModuleGetFunction)(&ctx->fnComposite, ctx->partitionModule, "simlod_composite_min"));
    CU(D(cuModuleGetFunction)(&ctx->fnPeerSignal, ctx->partitionModule, "simlod_peer_signal"));

    // buffers (main.cpp:552-586)
    SimlodBuffers& b = ctx->buf;
    b.momentary_bytes = config->momentary_bytes ? config->momentary_bytes : 300000000ull;
    b.nodes_bytes = config->nodes_bytes ? config->nodes_bytes : 40000000ull;
    b.renderbuffer_bytes = config->renderbuffer_bytes ? config->renderbuffer_bytes : 200000000ull;
    b.ring_bytes = RING_SLOTS * SLOT_POINTS * sizeof(SimlodPoint);
    uint64_t fbEnd = FB_OFFSET + (uint64_t)config->width * config->height * (8 + 4 + 16) + 64;
    if (fbEnd > b.renderbuffer_bytes) return fail(SIMLOD_ERR_INVALID, "render buffer too small for %ux%u", config->width, config->height);
    ALLOC(b.momentary, b.momentary_bytes);
    ALLOC(b.nodes, b.nodes_bytes);
    ALLOC(b.renderbuffer, b.renderbuffer_bytes);
    ALLOC(b.stats, sizeof(SimlodStats));
    CU(D(cuMemAlloc)(&ctx->numBatchesUploaded, 4));
    CU(D(cuMemAlloc)(&ctx->batchSizes, 4 * RING_SLOTS));
    CU(D(cuMemAlloc)(&ctx->frameStart, 8));
    CU(D(cuMemAlloc)(&ctx->scratch4, 16));
    CU(D(cuMemAlloc)(&ctx->cudaprint, 1024 * 1000 + 16));                 // CudaPrint ring (CudaPrint.cuh:33-36); never written
    CU(D(cuMemAlloc)(&ctx->flushBuf, L2_FLUSH_BYTES));
    CU(D(cuMemHostAlloc)((void**)&ctx->hStats, sizeof(SimlodStats), 0));
    CU(D(cuMemHostAlloc)((void**)&ctx->hStatsRing, 8 * sizeof(SimlodStats), 0));
    CU(D(cuMemHostAlloc)((void**)&ctx->hPublish, 16 * sizeof(SimlodContext::PublishMirror), 0));
    for (int i = 0; i < 16; i++) CU(D(cuEventCreate)(&ctx->evPublish[i], CU_EVENT_DISABLE_TIMING));
    for (int i = 0; i < 8; i++) CU(D(cuEventCreate)(&ctx->evStatsDone[i], CU_EVENT_DISABLE_TIMING));
    ALLOC(b.ring, b.ring_bytes);
    if (config->persistent_bytes) {
        b.persistent_bytes = config->persistent_bytes;
    } else {
        size_t freeMem = 0, totalMem = 0;
        CU(D(cuMemGetInfo)(&freeMem, &totalMem));
        b.persistent_bytes = (uint64_t)((double)freeMem * 0.80);
    }
    ALLOC(b.persistent, b.persistent_bytes);
    CU(D(cuMemsetD8)(b.momentary, 0, b.momentary_bytes));
    CU(D(cuMemsetD8)(b.nodes, 0, b.nodes_bytes));
    CU(D(cuMemsetD8)(b.stats, 0, sizeof(SimlodStats)));
    CU(D(cuMemsetD8)(ctx->numBatchesUploaded, 0, 4));
    CU(D(cuMemsetD8)(ctx->batchSizes, 0, 4 * RING_SLOTS));
    CU(D(cuMemsetD8)(ctx->cudaprint, 0, 16));

    // RGBA8 surface-capable array in place of the GL colour attachment (main.cpp:472-486)
    CUDA_ARRAY3D_DESCRIPTOR ad{};
    ad.Width = config->width; ad.Height = config->height; ad.Depth = 0;
    ad.Format = CU_AD_FORMAT_UNSIGNED_INT8; ad.NumChannels = 4; ad.Flags = CUDA_ARRAY3D_SURFACE_LDST;
    CU(D(cuArray3DCreate)(&ctx->colorArray, &ad));
    CUDA_RESOURCE_DESC rd{};
    rd.resType = CU_RESOURCE_TYPE_ARRAY; rd.res.array.hArray = ctx->colorArray;
    CU(D(cuSurfObjectCreate)(&ctx->surface, &rd));

    memset(&ctx->uniforms, 0, sizeof(ctx->uniforms));
    ctx->uniforms.width = (float)config->width;
    ctx->uniforms.height = (float)config->height;
    ctx->uniforms.persistentBufferCapacity = b.persistent_bytes;
    ctx->uniforms.momentaryBufferCapacity = b.momentary_bytes;
    int rc = computeGrids(ctx);
    if (rc != SIMLOD_OK) return rc;
    CU(D(cuCtxSynchronize)());
    return SIMLOD_OK;
}

int simlod_create(const SimlodConfig* config, SimlodContext** out) {
    if (!config || !out) return fail(SIMLOD_ERR_INVALID, "null argument");
    if (config->width == 0 || config->height == 0) return fail(SIMLOD_ERR_INVALID, "render target must be non-empty");
    if (config->renderbuffer_bytes && config->renderbuffer_bytes < 200000000ull)   // kernel_render lays its scratch out for the reference's 200 MB buffer (main.cpp:556)
        return fail(SIMLOD_ERR_INVALID, "renderbuffer_bytes %llu is below the 200 000 000 bytes the kernels are built for", (unsigned long long)config->renderbuffer_bytes);
    if (config->nodes_bytes && config->nodes_bytes < 40000000ull)     // kernel_construct's node capacity is the reference's 40 MB array (main.cpp:552-555)
        return fail(SIMLOD_ERR_INVALID, "nodes_bytes %llu is below the 40 000 000 bytes the kernels are built for", (unsigned long long)config->nodes_bytes);
    { int rc0 = loadDriver(); if (rc0) return rc0; }
    CU(D(cuInit)(0));
    SimlodContext* ctx = new SimlodContext();
    ctx->cfg = *config;
    // the primary context, so the library composes with other runtime-API users in the process
    CUresult r = D(cuDeviceGet)(&ctx->device, config->device);
    if (r != CUDA_SUCCESS) { delete ctx; return fail(SIMLOD_ERR_CUDA, "D(cuDeviceGet)(%d) failed: no such CUDA device", config->device); }
    r = D(cuDevicePrimaryCtxRetain)(&ctx->primary, ctx->device);
    if (r != CUDA_SUCCESS) { delete ctx; return fail(SIMLOD_ERR_CUDA, "cuDevicePrimaryCtxRetain failed on device %d", config->device); }
    int rc = createResources(ctx, config);
    if (rc != SIMLOD_OK) { simlod_destroy(ctx); return rc; }       // last_error keeps the reason
    *out = ctx;
    return SIMLOD_OK;
}

void simlod_destroy(SimlodContext* ctx) {
    if (!ctx) return;
    if (D(cuCtxSetCurrent)(ctx->primary) == CUDA_SUCCESS) {
        D(cuCtxSynchronize)();
        if (ctx->surface) D(cuSurfObjectDestroy)(ctx->surface);
        if (ctx->colorArray) D(cuArrayDestroy)(ctx->colorArray);
        CUdeviceptr ptrs[] = {ctx->buf.momentary, ctx->buf.nodes, ctx->buf.renderbuffer, ctx->buf.stats, ctx->buf.ring, ctx->buf.persistent,
                              ctx->numBatchesUploaded, ctx->batchSizes, ctx->frameStart, ctx->scratch4, ctx->cudaprint, ctx->flushBuf};
        for (CUdeviceptr p : ptrs) if (p) D(cuMemFree)(p);
        if (ctx->hStats) D(cuMemFreeHost)(ctx->hStats);
        if (ctx->hStatsRing) D(cuMemFreeHost)(ctx->hStatsRing);
        if (ctx->hPublish) D(cuMemFreeHost)(ctx->hPublish);
        for (int i = 0; i < 16; i++) if (ctx->evPublish[i]) D(cuEventDestroy)(ctx->evPublish[i]);
        for (int i = 0; i < 8; i++) if (ctx->evStatsDone[i]) D(cuEventDestroy)(ctx->evStatsDone[i]);
        for (int p = 0; p < 3; p++) if (ctx->programs[p].module) D(cuModuleUnload)(ctx->programs[p].module);
        if (ctx->utilModule) D(cuModuleUnload)(ctx->utilModule);
        if (ctx->partitionModule) D(cuModuleUnload)(ctx->partitionModule);
        if (ctx->partScratch) D(cuMemFree)(ctx->partScratch);
        if (ctx->lasModule) D(cuModuleUnload)(ctx->lasModule);
        if (ctx->genModule) D(cuModuleUnload)(ctx->genModule);
        if (ctx->lasStaging) D(cuMemFree)(ctx->lasStaging);
        delete ctx->loaderPool;          // joins the loader threads
        if (ctx->pinnedPool) D(cuMemFreeHost)(ctx->pinnedPool);
        for (int i = 0; i < 32; i++) if (ctx->evPool[i]) D(cuEventDestroy)(ctx->evPool[i]);
        if (ctx->evStart) D(cuEventDestroy)(ctx->evStart);
        if (ctx->evEnd) D(cuEventDestroy)(ctx->evEnd);
        if (ctx->evTotalStart) D(cuEventDestroy)(ctx->evTotalStart);
        if (ctx->evTotalEnd) D(cuEventDestroy)(ctx->evTotalEnd);
        for (int i = 0; i < 8; i++) for (int j = 0; j < 2; j++) if (ctx->evBurst[i][j]) D(cuEventDestroy)(ctx->evBurst[i][j]);
        for (uint64_t i = 0; i < RING_SLOTS; i++) if (ctx->evSlot[i]) D(cuEventDestroy)(ctx->evSlot[i]);
        if (ctx->streamMain) D(cuStreamDestroy)(ctx->streamMain);
        if (ctx->streamUpload) D(cuStreamDestroy)(ctx->streamUpload);
        D(cuDevicePrimaryCtxRelease)(ctx->device);
    }
    delete ctx;
}

int simlod_use_module(SimlodContext* ctx, int program, const char* cubin_path) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (program < 0 || program > 2) return fail(SIMLOD_ERR_INVALID, "unknown program %d", program);
    CU(D(cuCtxSynchronize)());
    if (!cubin_path) {
        rc = loadProgram(ctx, program, builtinImage(program), true);
    } else {
        std::ifstream f(cubin_path, std::ios::binary);
        if (!f) return fail(SIMLOD_ERR_MODULE, "cannot open %s", cubin_path);
        std::vector<char> image((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        image.push_back(0);
        rc = loadProgram(ctx, program, image.data(), false);
    }
    if (rc) return rc;
    return computeGrids(ctx);
}

int simlod_set_uniforms(SimlodContext* ctx, const SimlodUniforms* uniforms) {
    if (!ctx || !uniforms) return fail(SIMLOD_ERR_INVALID, "null argument");
    ctx->uniforms = *uniforms;
    ctx->uniforms.width = (float)ctx->cfg.width;                         // main.cpp:308-309
    ctx->uniforms.height = (float)ctx->cfg.height;
    ctx->uniforms.persistentBufferCapacity = ctx->buf.persistent_bytes;  // main.cpp:325-326
    ctx->uniforms.momentaryBufferCapacity = ctx->buf.momentary_bytes;
    return SIMLOD_OK;
}

int simlod_get_uniforms(SimlodContext* ctx, SimlodUniforms* out) {
    if (!ctx || !out) return fail(SIMLOD_ERR_INVALID, "null argument");
    *out = ctx->uniforms;
    return SIMLOD_OK;
}

int simlod_reset(SimlodContext* ctx) {
    // The reference launches the reset kernel with 1 block x 1 thread (main.cpp:348-354); one thread then zeroes the
    // root's 256 KiB grid alone. The kernel is grid-stride (reference reset.cu:78-85 and ours), so the
    // launch surface gives it one block per SM; simlod_reset_with_grid(ctx, 1, 1) is the reference's shape.
    if (!ctx) return fail(SIMLOD_ERR_INVALID, "null context");
    return simlod_reset_with_grid(ctx, (uint32_t)ctx->numSMs, 256);
}

int simlod_reset_with_grid(SimlodContext* ctx, uint32_t blocks, uint32_t threads) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (blocks == 0 || threads == 0 || threads > 1024) return fail(SIMLOD_ERR_INVALID, "bad reset launch shape %u x %u", blocks, threads);
    CU(D(cuStreamSynchronize)(ctx->streamUpload));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    CU(D(cuMemsetD8Async)(ctx->buf.nodes, 0, ctx->buf.nodes_bytes, ctx->streamMain));
    SimlodUniforms u = ctx->uniforms;
    u.frameCounter = ctx->frameCounter;
    CUdeviceptr persistent = ctx->buf.persistent, nodes = ctx->buf.nodes, stats = ctx->buf.stats, cudaprint = ctx->cudaprint,
                nbu = ctx->numBatchesUploaded, bs = ctx->batchSizes;
    void* args[] = {&u, &persistent, &nodes, &stats, &cudaprint, &nbu, &bs};      // main.cpp:337-345
    CU(D(cuLaunchCooperativeKernel)(ctx->programs[SIMLOD_PROGRAM_RESET].fn, blocks, 1, 1, threads, 1, 1, 0, ctx->streamMain, args));
    ctx->launches++;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    ctx->uploaded = 0;
    ctx->processed = 0;
    ctx->unpublished = 0;
    memset(ctx->hostSizes, 0, sizeof(ctx->hostSizes));
    return SIMLOD_OK;
}

static int uploadCommon(SimlodContext* ctx, const void* host, CUdeviceptr dev, uint32_t count, bool publish = true) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (count > SLOT_POINTS) return fail(SIMLOD_ERR_INVALID, "batch of %u points exceeds the ring slot size of %llu", count, (unsigned long long)SLOT_POINTS);
    if (ctx->uploaded - ctx->processed >= RING_SLOTS) {
        rc = readStats(ctx); if (rc) return rc;
        if (ctx->uploaded - ctx->processed >= RING_SLOTS) return fail(SIMLOD_ERR_RING_FULL, "all %llu ring slots hold unprocessed batches", (unsigned long long)RING_SLOTS);
    }
    uint32_t slot = ctx->uploaded % RING_SLOTS;
    CUdeviceptr dst = ctx->buf.ring + (uint64_t)slot * SLOT_POINTS * sizeof(SimlodPoint);
    if (count) {
        if (host) CU(D(cuMemcpyHtoDAsync)(dst, host, (size_t)count * sizeof(SimlodPoint), ctx->streamUpload));   // main.cpp:1040
        else      CU(D(cuMemcpyDtoDAsync)(dst, dev, (size_t)count * sizeof(SimlodPoint), ctx->streamUpload));
    }
    if (publish) return publishBatch(ctx, slot, count);
    ctx->hostSizes[slot] = count;           // published with its group: publishPending()
    ctx->uploaded++;
    ctx->unpublished++;
    return SIMLOD_OK;
}

int simlod_upload_batch(SimlodContext* ctx, const SimlodPoint* host_points, uint32_t count) {
    if (!host_points && count) return fail(SIMLOD_ERR_INVALID, "null points");
    return uploadCommon(ctx, host_points, 0, count);
}
int simlod_upload_batch_device(SimlodContext* ctx, uint64_t device_points, uint32_t count) {
    if (!device_points && count) return fail(SIMLOD_ERR_INVALID, "null points");
    return uploadCommon(ctx, nullptr, (CUdeviceptr)device_points, count);
}

static int uploadLasCommon(SimlodContext* ctx, const void* host, CUdeviceptr dev, uint32_t count, const SimlodLasLayout* layout) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!layout) return fail(SIMLOD_ERR_INVALID, "null layout");
    if (count > SLOT_POINTS) return fail(SIMLOD_ERR_INVALID, "batch of %u points exceeds the ring slot size of %llu", count, (unsigned long long)SLOT_POINTS);
    if (layout->bytes_per_point < 12 || layout->bytes_per_point > 96) return fail(SIMLOD_ERR_INVALID, "unsupported LAS record size %u", layout->bytes_per_point);
    uint32_t offsetRgb = 0;                                   // LasLoader.cpp:179-188
    if (layout->format == 2) offsetRgb = 20; else if (layout->format == 3) offsetRgb = 28;
    if (layout->format == 5) offsetRgb = 28;
    if (layout->format == 7) offsetRgb = 30;
    if (offsetRgb && offsetRgb + 6 > layout->bytes_per_point) return fail(SIMLOD_ERR_INVALID, "LAS format %u does not fit %u-byte records", layout->format, layout->bytes_per_point);
    if (ctx->uploaded - ctx->processed >= RING_SLOTS) {
        rc = readStats(ctx); if (rc) return rc;
        if (ctx->uploaded - ctx->processed >= RING_SLOTS) return fail(SIMLOD_ERR_RING_FULL, "all %llu ring slots hold unprocessed batches", (unsigned long long)RING_SLOTS);
    }
    uint32_t slot = ctx->uploaded % RING_SLOTS;
    CUdeviceptr dst = ctx->buf.ring + (uint64_t)slot * SLOT_POINTS * sizeof(SimlodPoint);
    if (count) {
        CUdeviceptr records = dev;
        if (host) {
            if (!ctx->lasStaging) CU(D(cuMemAlloc)(&ctx->lasStaging, (size_t)SLOT_POINTS * 96));
            records = ctx->lasStaging;                        // reused batch after batch: copy and decode are ordered by the upload stream
            CU(D(cuMemcpyHtoDAsync)(records, host, (size_t)count * layout->bytes_per_point, ctx->streamUpload));
        }
        uint64_t numPoints = count;
        uint32_t bpp = layout->bytes_per_point;
        double sx = layout->scale[0], sy = layout->scale[1], sz = layout->scale[2];
        double ox = layout->offset[0] + layout->translation[0], oy = layout->offset[1] + layout->translation[1], oz = layout->offset[2] + layout->translation[2];   // LasLoader.cpp:199-201
        void* args[] = {&records, &numPoints, &bpp, &offsetRgb, &sx, &sy, &sz, &ox, &oy, &oz, &dst};
        unsigned blocks = (unsigned)std::min<uint64_t>((count + 255) / 256, (uint64_t)ctx->numSMs * 8);
        CU(D(cuLaunchKernel)(ctx->fnLas, blocks, 1, 1, 256, 1, 1, 0, ctx->streamUpload, args, nullptr));
        ctx->launches++;
    }
    return publishBatch(ctx, slot, count);
}

int simlod_upload_batch_las(SimlodContext* ctx, const void* host_records, uint32_t count, const SimlodLasLayout* layout) {
    if (!host_records && count) return fail(SIMLOD_ERR_INVALID, "null records");
    return uploadLasCommon(ctx, host_records, 0, count, layout);
}
int simlod_upload_batch_las_device(SimlodContext* ctx, uint64_t device_records, uint32_t count, const SimlodLasLayout* layout) {
    if (!device_records && count) return fail(SIMLOD_ERR_INVALID, "null records");
    return uploadLasCommon(ctx, nullptr, (CUdeviceptr)device_records, count, layout);
}

int simlod_update_octree(SimlodContext* ctx, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    rc = launchConstruct(ctx, kernel_ms); if (rc) return rc;
    rc = readStats(ctx); if (rc) return rc;
    return checkOverflow(ctx);
}

// The main loop's streaming behaviour (main.cpp:1176-1180 + the uploader thread, :963-1063) without a frame in between:
// uploads run ahead as far as the 50-slot ring allows, update launches are enqueued back to back (each consumes at most
// 20 batches or 10 ms, voxels.cu:22,883,940), and the host learns what the device has consumed from asynchronous Stats
// snapshots (one per launch, as the reference copies Stats every frame, main.cpp:1201-1216) — it never drains the
// launch stream to decide what to do next, so the GPU does not idle between launches.
static int insertCommon(SimlodContext* ctx, const SimlodPoint* host, CUdeviceptr dev, uint64_t count, float* kernel_ms, float* total_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    const uint64_t numBatches = (count + SLOT_POINTS - 1) / SLOT_POINTS;
    rc = readStats(ctx); if (rc) return rc;
    const uint32_t target = ctx->uploaded + (uint32_t)numBatches;
    uint64_t next = 0;
    float total = 0.0f;
    // A launch starts once the batches it is meant to consume are published (stream wait on the slot's event) instead of
    // snapshotting a half-filled ring. Device-resident sources arrive far faster than they are consumed: full 20-batch
    // launches. Host sources arrive at PCIe speed, slower than the builder: launch from 2 batches on, so that
    // insertion trails the upload closely.
    const uint32_t gate = host ? 2u : 20u;
    int inFlight[8]; int numInFlight = 0, nextSlot = 0;      // FIFO of launch slots whose Stats snapshot is pending
    uint32_t covered = ctx->processed;                       // batches the enqueued launches are expected to have consumed
    uint32_t stalled = 0;
    auto drainOne = [&](bool block) -> int {                 // 1: a snapshot was taken in, 0: none ready, < 0: error
        if (numInFlight == 0) return 0;
        const int k = inFlight[0];
        if (!block) {
            CUresult q = D(cuEventQuery)(ctx->evStatsDone[k]);
            if (q == CUDA_ERROR_NOT_READY) return 0;
            if (q != CUDA_SUCCESS) return fail(SIMLOD_ERR_CUDA, "event query failed (%d)", (int)q);
        } else {
            CUresult q = D(cuEventSynchronize)(ctx->evStatsDone[k]);
            if (q != CUDA_SUCCESS) { const char* e = nullptr; D(cuGetErrorString)(q, &e); return fail(SIMLOD_ERR_CUDA, "kernel_construct failed: %s (%d)", e ? e : "?", (int)q); }
        }
        float ms = 0.0f;
        D(cuEventElapsedTime)(&ms, ctx->evBurst[k][0], ctx->evBurst[k][1]);
        total += ms;
        const uint32_t before = ctx->processed;
        *ctx->hStats = ctx->hStatsRing[k];
        ctx->processed = ctx->hStats->batchletIndex;
        for (int i = 1; i < numInFlight; i++) inFlight[i - 1] = inFlight[i];
        numInFlight--;
        if (ctx->hStats->memCapacityReached) return fail(SIMLOD_ERR_CAPACITY, "persistent heap almost full after %llu points", (unsigned long long)ctx->hStats->numPointsProcessed);
        int orc = checkOverflow(ctx); if (orc) return orc;
        stalled = ctx->processed == before ? stalled + 1 : 0;
        if (numInFlight == 0 && covered > ctx->processed) covered = ctx->processed;     // a launch ran into its 10 ms budget: the rest is launched again
        return 1;
    };
    CU(D(cuEventRecord)(ctx->evTotalStart, ctx->streamMain));
    while (ctx->processed < target) {
        bool progress = false;
        // uploader: keep the ring as full as back-pressure allows (main.cpp:1012,1033-1056)
        while (next < numBatches && ctx->uploaded - ctx->processed < RING_SLOTS) {
            uint64_t first = next * SLOT_POINTS;
            uint32_t n = (uint32_t)std::min<uint64_t>(SLOT_POINTS, count - first);
            rc = uploadCommon(ctx, host ? host + first : nullptr, dev ? dev + first * sizeof(SimlodPoint) : 0, n, false);
            if (rc) return rc;
            next++;
            progress = true;
            if (host && ctx->unpublished >= gate) { rc = publishPending(ctx); if (rc) return rc; }      // a host source trickles in at PCIe speed: publish as it goes
        }
        rc = publishPending(ctx); if (rc) return rc;
        while (numInFlight < 8 && ctx->uploaded > covered && (ctx->uploaded - covered >= gate || next == numBatches)) {
            const uint32_t take = std::min<uint32_t>(20u, ctx->uploaded - covered);
            CU(D(cuStreamWaitEvent)(ctx->streamMain, ctx->evSlot[(covered + take - 1u) % RING_SLOTS], 0));
            const int k = nextSlot; nextSlot = (nextSlot + 1) % 8;
            rc = enqueueConstruct(ctx, k); if (rc) return rc;
            CU(D(cuMemcpyDtoHAsync)(&ctx->hStatsRing[k], ctx->buf.stats, sizeof(SimlodStats), ctx->streamMain));
            CU(D(cuEventRecord)(ctx->evStatsDone[k], ctx->streamMain));
            inFlight[numInFlight++] = k;
            covered += take;
            progress = true;
        }
        for (;;) {
            int d = drainOne(false);
            if (d < 0) return d;
            if (d == 0) break;
            progress = true;
        }
        if (!progress) {
            if (numInFlight > 0) { int d = drainOne(true); if (d < 0) return d; }
            else if (stalled > 4) return fail(SIMLOD_ERR_CUDA, "kernel_construct makes no progress (%u of %u batches consumed)", ctx->processed, target);
            else covered = ctx->processed;
        }
    }
    while (numInFlight > 0) { int d = drainOne(true); if (d < 0) return d; }
    CU(D(cuEventRecord)(ctx->evTotalEnd, ctx->streamMain));
    CU(D(cuEventSynchronize)(ctx->evTotalEnd));
    if (kernel_ms) *kernel_ms = total;
    if (total_ms) CU(D(cuEventElapsedTime)(total_ms, ctx->evTotalStart, ctx->evTotalEnd));
    return SIMLOD_OK;
}

// Device-resident source: the point set already IS a sequence of 1 000 000-point batches in HBM, so copying it into the
// ring would only move 16 B/point a second time — and those device-to-device copies cannot run under the persistent
// cooperative kernel (measured: every launch waited 0.24 ms for the 20 copies behind it, tools/launch_gaps.py).
// kernel_construct addresses batch g as points + (g % 50) * 1 000 000 (voxels.cu:886-889); within one window of 50
// consecutive batches that is a linear map of g, so the launches of a window get a `points` argument that makes slot
// g % 50 land on batch g of the caller's buffer. The ring protocol is unchanged from the kernel's side (sizes and counter are
// published per window, the next window only after the device has consumed the current one); only the bytes do not move.
static int insertDeviceDirect(SimlodContext* ctx, CUdeviceptr dev, uint64_t count, float* kernel_ms, float* total_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    const uint64_t numBatches = (count + SLOT_POINTS - 1) / SLOT_POINTS;
    rc = readStats(ctx); if (rc) return rc;
    while (ctx->processed < ctx->uploaded) {               // batches uploaded earlier sit in the real ring: consume them first
        rc = launchConstruct(ctx, nullptr); if (rc) return rc;
        rc = readStats(ctx); if (rc) return rc;
        if (ctx->hStats->memCapacityReached) return fail(SIMLOD_ERR_CAPACITY, "persistent heap almost full after %llu points", (unsigned long long)ctx->hStats->numPointsProcessed);
    }
    const uint32_t g0 = ctx->uploaded;                     // global index of this call's first batch
    const uint32_t target = g0 + (uint32_t)numBatches;
    float total = 0.0f;
    int inFlight[8]; int numInFlight = 0, nextSlot = 0;
    uint32_t covered = ctx->processed, stalled = 0;
    CUdeviceptr base = 0;
    CU(D(cuEventRecord)(ctx->evTotalStart, ctx->streamMain));
    while (ctx->processed < target) {
        if (numInFlight == 0) {
            covered = ctx->processed;
            if (ctx->uploaded == ctx->processed) {         // the window is consumed: publish the next one (sizes + counter only)
                const uint32_t window = ctx->processed / (uint32_t)RING_SLOTS;
                const uint32_t windowEnd = std::min<uint32_t>(target, (window + 1u) * (uint32_t)RING_SLOTS);
                while (ctx->uploaded < windowEnd) {
                    const uint64_t first = (uint64_t)(ctx->uploaded - g0) * SLOT_POINTS;
                    ctx->hostSizes[ctx->uploaded % RING_SLOTS] = (uint32_t)std::min<uint64_t>(SLOT_POINTS, count - first);
                    ctx->uploaded++;
                    ctx->unpublished++;
                }
                rc = publishPending(ctx); if (rc) return rc;
                // slot s of this window = batch window * 50 + s = the caller's batch (window * 50 + s - g0)
                base = dev + (uint64_t)((int64_t)window * (int64_t)RING_SLOTS - (int64_t)g0) * (SLOT_POINTS * sizeof(SimlodPoint));
            }
            if (stalled > 4) return fail(SIMLOD_ERR_CUDA, "kernel_construct makes no progress (%u of %u batches consumed)", ctx->processed, target);
            while (numInFlight < 8 && ctx->uploaded > covered) {
                const uint32_t take = std::min<uint32_t>(20u, ctx->uploaded - covered);
                CU(D(cuStreamWaitEvent)(ctx->streamMain, ctx->evSlot[(covered + take - 1u) % RING_SLOTS], 0));
                const int k = nextSlot; nextSlot = (nextSlot + 1) % 8;
                rc = enqueueConstruct(ctx, k, base); if (rc) return rc;
                CU(D(cuMemcpyDtoHAsync)(&ctx->hStatsRing[k], ctx->buf.stats, sizeof(SimlodStats), ctx->streamMain));
                CU(D(cuEventRecord)(ctx->evStatsDone[k], ctx->streamMain));
                inFlight[numInFlight++] = k;
                covered += take;
            }
        }
        const int k = inFlight[0];
        CUresult q = D(cuEventSynchronize)(ctx->evStatsDone[k]);
        if (q != CUDA_SUCCESS) { const char* e = nullptr; D(cuGetErrorString)(q, &e); return fail(SIMLOD_ERR_CUDA, "kernel_construct failed: %s (%d)", e ? e : "?", (int)q); }
        float ms = 0.0f;
        D(cuEventElapsedTime)(&ms, ctx->evBurst[k][0], ctx->evBurst[k][1]);
        total += ms;
        const uint32_t before = ctx->processed;
        *ctx->hStats = ctx->hStatsRing[k];
        ctx->processed = ctx->hStats->batchletIndex;
        for (int i = 1; i < numInFlight; i++) inFlight[i - 1] = inFlight[i];
        numInFlight--;
        stalled = ctx->processed == before ? stalled + 1 : 0;
        if (ctx->hStats->memCapacityReached) return fail(SIMLOD_ERR_CAPACITY, "persistent heap almost full after %llu points", (unsigned long long)ctx->hStats->numPointsProcessed);
        rc = checkOverflow(ctx); if (rc) return rc;
    }
    CU(D(cuEventRecord)(ctx->evTotalEnd, ctx->streamMain));
    CU(D(cuEventSynchronize)(ctx->evTotalEnd));
    if (kernel_ms) *kernel_ms = total;
    if (total_ms) CU(D(cuEventElapsedTime)(total_ms, ctx->evTotalStart, ctx->evTotalEnd));
    return SIMLOD_OK;
}

int simlod_insert(SimlodContext* ctx, const SimlodPoint* host_points, uint64_t count, float* kernel_ms, float* total_ms) {
    if (!host_points && count) return fail(SIMLOD_ERR_INVALID, "null points");
    return insertCommon(ctx, host_points, 0, count, kernel_ms, total_ms);
}
int simlod_insert_device(SimlodContext* ctx, uint64_t device_points, uint64_t count, float* kernel_ms, float* total_ms) {
    if (!device_points && count) return fail(SIMLOD_ERR_INVALID, "null points");
    if (!ctx) return fail(SIMLOD_ERR_INVALID, "null context");
    if ((device_points & 15ull) != 0 || getenv("SIMLOD_NO_DIRECT") != nullptr) return insertCommon(ctx, nullptr, (CUdeviceptr)device_points, count, kernel_ms, total_ms);    // unaligned source: through the ring
    return insertDeviceDirect(ctx, (CUdeviceptr)device_points, count, kernel_ms, total_ms);
}

// ---- streaming front end (SURVEY.md §8f-1) -------------------------------------------------------------
int simlod_insert_simlod_file(SimlodContext* ctx, const char* path, int loader_threads, uint64_t* num_points,
                              float* kernel_ms, float* total_ms) {
    return simlod_insert_simlod_file_ex(ctx, path, loader_threads, 0, num_points, kernel_ms, total_ms);
}

int simlod_insert_simlod_file_ex(SimlodContext* ctx, const char* path, int loader_threads, uint32_t flags, uint64_t* num_points,
                                 float* kernel_ms, float* total_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!path) return fail(SIMLOD_ERR_INVALID, "null path");
    const bool direct = (flags & SIMLOD_STREAM_DIRECT) != 0;
    constexpr int POOL_SLOTS = 32;         // 512 MB page-locked (the reference: 200 x 16 MB, main.cpp:35)
    const uint64_t slotBytes = SLOT_POINTS * sizeof(SimlodPoint);
    FILE* f = fopen(path, "rb");
    if (!f) return fail(SIMLOD_ERR_INVALID, "cannot open %s", path);
    float hdr[6];
    size_t got = fread(hdr, 1, sizeof(hdr), f);
    fseek(f, 0, SEEK_END);
    const uint64_t fileSize = (uint64_t)ftell(f);
    fclose(f);
    if (got != sizeof(hdr) || fileSize < 24) return fail(SIMLOD_ERR_INVALID, "%s is not a .simlod file", path);
    const uint64_t numPoints = (fileSize - 24) / 16;                       // main.cpp:738
    const uint64_t numBatches = (numPoints + SLOT_POINTS - 1) / SLOT_POINTS;
    if (num_points) *num_points = numPoints;
    for (int i = 0; i < 3; i++) { ctx->uniforms.boxMin[i] = 0.0f; ctx->uniforms.boxMax[i] = hdr[3 + i] - hdr[i]; }   // main.cpp:312-313
    rc = simlod_reset(ctx); if (rc) return rc;                            // reload() -> reset
    if (!ctx->pinnedPool) {
        NumaLocal onGpuNode(ctx);
        CU(D(cuMemHostAlloc)(&ctx->pinnedPool, (size_t)POOL_SLOTS * slotBytes, CU_MEMHOSTALLOC_PORTABLE));
        for (int i = 0; i < POOL_SLOTS; i++) CU(D(cuEventCreate)(&ctx->evPool[i], CU_EVENT_DISABLE_TIMING));
    }
    // loaders: batch k goes to pool slot k % POOL_SLOTS once the copy of batch k - POOL_SLOTS has left it. The unit
    // of work is a 1 MB piece of a batch, handed out in file order, so that all threads read the batch the uploader
    // needs next (the reference reads one whole batch per thread, main.cpp:811-958: every batch then arrives late).
    constexpr uint64_t PIECE_POINTS = 65536, PIECES = (SLOT_POINTS + PIECE_POINTS - 1) / PIECE_POINTS;
    const bool trace = getenv("SIMLOD_STREAM_TRACE") != nullptr;          // developer aid: host timeline to stderr
    const auto tBegin = std::chrono::steady_clock::now();
    auto since = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tBegin).count(); };
    double tSpawned = 0, tFirst = 0, tAllLoaded = 0, tLastUpload = 0;
    std::vector<std::atomic<int>> loaded(numBatches);          // pieces of batch k that have arrived
    for (auto& l : loaded) l.store(0);
    std::atomic<int64_t> copiesDone{0};           // batches whose host->device copy has completed
    std::atomic<uint64_t> nextPiece{0};
    std::atomic<bool> abort{false};
    const int nThreads = std::max(1, std::min(loader_threads, 64));
    // SIMLOD_STREAM_DIRECT: unbuffered reads, as the reference's Windows loader does (SimlodLoader.cpp:59-141, FILE_FLAG_NO_BUFFERING):
    // whole 4 KB blocks straight from the device into a per-thread block buffer — no page-cache copy, no cache pollution —
    // for files that are not resident in the page cache (a cold 5.6 GB scan gains nothing from being cached on the way)
    const int fd = open(path, direct ? (O_RDONLY | O_DIRECT) : O_RDONLY);
    if (fd < 0) return fail(SIMLOD_ERR_INVALID, direct ? "cannot open %s with O_DIRECT (tmpfs and some overlay file systems do not support it)" : "cannot open %s", path);
    if (!ctx->loaderPool) ctx->loaderPool = new LoaderPool();
    LoaderPool* pool = ctx->loaderPool;
    pool->run(nThreads, [&, pool](int worker) {
        for (;;) {
            const uint64_t item = nextPiece.fetch_add(1);
            const uint64_t k = item / PIECES, piece = item % PIECES;
            if (k >= numBatches || abort.load()) break;
            while (copiesDone.load() + POOL_SLOTS <= (int64_t)k && !abort.load()) std::this_thread::yield();
            const uint64_t inBatch = std::min<uint64_t>(SLOT_POINTS, numPoints - k * SLOT_POINTS);
            const uint64_t p0 = piece * PIECE_POINTS;
            if (p0 < inBatch) {
                uint64_t bytes = std::min<uint64_t>(PIECE_POINTS, inBatch - p0) * 16;
                char* dst = (char*)ctx->pinnedPool + (k % POOL_SLOTS) * slotBytes + p0 * 16;
                off_t at = (off_t)(24 + (k * SLOT_POINTS + p0) * 16);
                if (direct) {
                    // the piece is <= 1 MB of records at a file offset that is 8 (mod 16): read the 4 KB blocks that cover it
                    char* blockBuf = pool->directBuffer(worker);
                    const off_t a0 = at & ~(off_t)4095;
                    const size_t want = (size_t)((((uint64_t)at + bytes + 4095ull) & ~4095ull) - (uint64_t)a0);
                    size_t have = 0;
                    while (have < want) {
                        ssize_t r = pread(fd, blockBuf + have, want - have, a0 + (off_t)have);
                        if (r < 0) { abort.store(true); break; }
                        if (r == 0) break;                                        // end of file inside the last block
                        have += (size_t)r;
                        if (r % 4096) break;                                      // short read at the end of the file
                    }
                    if (have < (size_t)(at - a0) + bytes) abort.store(true);
                    else copyStreamingU(dst, blockBuf + (at - a0), bytes);
                    bytes = 0;
                }
                char* stage = pool->bounce[worker];
                while (bytes) {
                    uint64_t want = std::min<uint64_t>(bytes, LoaderPool::BOUNCE_BYTES), have = 0;
                    while (have < want) {
                        ssize_t r = pread(fd, stage + have, want - have, at + (off_t)have);
                        if (r <= 0) { abort.store(true); break; }
                        have += (uint64_t)r;
                    }
                    if (have < want) break;
                    copyStreaming(dst, stage, want);
                    dst += want; at += (off_t)want; bytes -= want;
                }
            }
            loaded[k].fetch_add(1);
        }
    });
    const int allPieces = (int)PIECES;
    tSpawned = since();
    auto joinAll = [&]() { abort.store(true); ctx->loaderPool->wait(); close(fd); };

    float kernelTotal = 0.0f;
    int pairInUse[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int nextPair = 0;
    auto launch = [&](uint32_t lastWanted) -> int {
        int k = nextPair; nextPair = (nextPair + 1) % 8;
        if (pairInUse[k]) {            // the launch that used this pair is 8 launches old: collect its time
            CUresult r = D(cuEventSynchronize)(ctx->evBurst[k][1]);
            if (r != CUDA_SUCCESS) return fail(SIMLOD_ERR_CUDA, "event sync failed");
            float ms = 0.0f; D(cuEventElapsedTime)(&ms, ctx->evBurst[k][0], ctx->evBurst[k][1]); kernelTotal += ms;
        }
        CUresult r = D(cuStreamWaitEvent)(ctx->streamMain, ctx->evSlot[lastWanted % RING_SLOTS], 0);
        if (r != CUDA_SUCCESS) return fail(SIMLOD_ERR_CUDA, "stream wait failed");
        int lrc = enqueueConstruct(ctx, k);
        pairInUse[k] = 1;
        return lrc;
    };

    rc = readStats(ctx); if (rc) { joinAll(); return rc; }
    const uint32_t firstUploaded = ctx->uploaded;
    CUresult cr = D(cuEventRecord)(ctx->evTotalStart, ctx->streamMain);
    if (cr != CUDA_SUCCESS) { joinAll(); return fail(SIMLOD_ERR_CUDA, "event record failed"); }
    int64_t copiesEnqueued = 0;
    for (uint64_t k = 0; k < numBatches; k++) {
        while (loaded[k].load() < allPieces && !abort.load()) std::this_thread::yield();
        if (abort.load()) { joinAll(); return fail(SIMLOD_ERR_INVALID, "read error in %s", path); }
        if (k == 0) tFirst = since();
        if (k + 1 == numBatches) tAllLoaded = since();
        // back-pressure (main.cpp:1012): when the ring is full, launch until a slot frees (or the device stops consuming)
        while (ctx->uploaded - ctx->processed >= RING_SLOTS - 1) {
            rc = readStats(ctx); if (rc) { joinAll(); return rc; }
            if (ctx->uploaded - ctx->processed < RING_SLOTS - 1) break;
            if (ctx->hStats->memCapacityReached) { joinAll(); return fail(SIMLOD_ERR_CAPACITY, "persistent heap almost full after %llu points", (unsigned long long)ctx->hStats->numPointsProcessed); }
            rc = checkOverflow(ctx); if (rc) { joinAll(); return rc; }
            rc = launch(ctx->uploaded - 1); if (rc) { joinAll(); return rc; }
        }
        uint64_t first = k * SLOT_POINTS;
        uint32_t n = (uint32_t)std::min<uint64_t>(SLOT_POINTS, numPoints - first);
        const SimlodPoint* src = (const SimlodPoint*)((char*)ctx->pinnedPool + (k % POOL_SLOTS) * slotBytes);
        rc = uploadCommon(ctx, src, 0, n); if (rc) { joinAll(); return rc; }
        cr = D(cuEventRecord)(ctx->evPool[k % POOL_SLOTS], ctx->streamUpload);
        if (cr != CUDA_SUCCESS) { joinAll(); return fail(SIMLOD_ERR_CUDA, "event record failed"); }
        copiesEnqueued++;
        // pool slots whose copy has completed are handed back to the loaders (in order)
        while (copiesDone.load() < copiesEnqueued && D(cuEventQuery)(ctx->evPool[copiesDone.load() % POOL_SLOTS]) == CUDA_SUCCESS) copiesDone.fetch_add(1);
        if ((k & 1) == 1 || k + 1 == numBatches) { rc = launch(ctx->uploaded - 1); if (rc) { joinAll(); return rc; } }
        // when all pool slots are in flight, wait for the oldest copy instead of spinning on the loaders
        if (copiesEnqueued - copiesDone.load() >= POOL_SLOTS) {
            D(cuEventSynchronize)(ctx->evPool[copiesDone.load() % POOL_SLOTS]);
            while (copiesDone.load() < copiesEnqueued && D(cuEventQuery)(ctx->evPool[copiesDone.load() % POOL_SLOTS]) == CUDA_SUCCESS) copiesDone.fetch_add(1);
        }
    }
    tLastUpload = since();
    ctx->loaderPool->wait();
    close(fd);
    const double tJoined = since();
    // drain: launches until every batch has been consumed
    const uint32_t target = firstUploaded + (uint32_t)numBatches;
    rc = readStats(ctx); if (rc) return rc;
    while (ctx->processed < target) {
        rc = launch(ctx->uploaded - 1); if (rc) return rc;
        rc = readStats(ctx); if (rc) return rc;
        if (ctx->hStats->memCapacityReached) return fail(SIMLOD_ERR_CAPACITY, "persistent heap almost full after %llu points", (unsigned long long)ctx->hStats->numPointsProcessed);
        rc = checkOverflow(ctx); if (rc) return rc;
    }
    CU(D(cuEventRecord)(ctx->evTotalEnd, ctx->streamMain));
    CU(D(cuEventSynchronize)(ctx->evTotalEnd));
    for (int k = 0; k < 8; k++) if (pairInUse[k]) { float ms = 0.0f; D(cuEventElapsedTime)(&ms, ctx->evBurst[k][0], ctx->evBurst[k][1]); kernelTotal += ms; }
    if (kernel_ms) *kernel_ms = kernelTotal;
    if (total_ms) CU(D(cuEventElapsedTime)(total_ms, ctx->evTotalStart, ctx->evTotalEnd));
    if (trace) fprintf(stderr, "[simlod stream] %llu batches, %d threads: started %.2f ms, first batch %.2f, all loaded %.2f, last upload enqueued %.2f, loaders idle %.2f, done %.2f\n",
                       (unsigned long long)numBatches, nThreads, tSpawned, tFirst, tAllLoaded, tLastUpload, tJoined, since());
    return SIMLOD_OK;
}

int simlod_render(SimlodContext* ctx, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    SimlodUniforms u = ctx->uniforms;
    u.frameCounter = ctx->frameCounter++;
    CUdeviceptr rb = ctx->buf.renderbuffer, nodes = ctx->buf.nodes, stats = ctx->buf.stats, frameStart = ctx->frameStart, cudaprint = ctx->cudaprint;
    CUsurfObject surf = ctx->surface;
    void* args[] = {&rb, &u, &nodes, &surf, &stats, &frameStart, &cudaprint};     // main.cpp:499-507
    CU(D(cuEventRecord)(ctx->evStart, ctx->streamMain));
    CU(D(cuLaunchCooperativeKernel)(ctx->programs[SIMLOD_PROGRAM_RENDER].fn, ctx->renderBlocks, 1, 1, 256, 1, 1, 0, ctx->streamMain, args));
    CU(D(cuEventRecord)(ctx->evEnd, ctx->streamMain));
    ctx->launches++;
    CU(D(cuEventSynchronize)(ctx->evEnd));
    if (kernel_ms) CU(D(cuEventElapsedTime)(kernel_ms, ctx->evStart, ctx->evEnd));
    return SIMLOD_OK;
}

int simlod_get_stats(SimlodContext* ctx, SimlodStats* out) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!out) return fail(SIMLOD_ERR_INVALID, "null argument");
    rc = readStats(ctx); if (rc) return rc;
    *out = *ctx->hStats;
    return SIMLOD_OK;
}

int simlod_read_framebuffer(SimlodContext* ctx, uint64_t* out) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!out) return fail(SIMLOD_ERR_INVALID, "null argument");
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    CU(D(cuMemcpyDtoH)(out, ctx->buf.renderbuffer + FB_OFFSET, (size_t)ctx->cfg.width * ctx->cfg.height * 8));
    return SIMLOD_OK;
}

int simlod_read_surface(SimlodContext* ctx, uint32_t* out) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!out) return fail(SIMLOD_ERR_INVALID, "null argument");
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    CUDA_MEMCPY2D cp{};
    cp.srcMemoryType = CU_MEMORYTYPE_ARRAY; cp.srcArray = ctx->colorArray;
    cp.dstMemoryType = CU_MEMORYTYPE_HOST; cp.dstHost = out; cp.dstPitch = (size_t)ctx->cfg.width * 4;
    cp.WidthInBytes = (size_t)ctx->cfg.width * 4; cp.Height = ctx->cfg.height;
    CU(D(cuMemcpy2D)(&cp));
    return SIMLOD_OK;
}

int simlod_get_buffers(SimlodContext* ctx, SimlodBuffers* out) {
    if (!ctx || !out) return fail(SIMLOD_ERR_INVALID, "null argument");
    *out = ctx->buf;
    return SIMLOD_OK;
}

int simlod_memcpy_dtoh(SimlodContext* ctx, void* dst, uint64_t src_device, uint64_t bytes) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    CU(D(cuMemcpyDtoH)(dst, (CUdeviceptr)src_device, (size_t)bytes));
    return SIMLOD_OK;
}
int simlod_memcpy_htod(SimlodContext* ctx, uint64_t dst_device, const void* src, uint64_t bytes) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    CU(D(cuMemcpyHtoD)((CUdeviceptr)dst_device, src, (size_t)bytes));
    return SIMLOD_OK;
}

int simlod_host_alloc(SimlodContext* ctx, uint64_t bytes, void** out) {
    int rc = setCurrent(ctx); if (rc) return rc;
    NumaLocal onGpuNode(ctx);
    CU(D(cuMemHostAlloc)(out, (size_t)bytes, CU_MEMHOSTALLOC_PORTABLE));
    return SIMLOD_OK;
}
int simlod_host_free(SimlodContext* ctx, void* ptr) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CU(D(cuMemFreeHost)(ptr));
    return SIMLOD_OK;
}
int simlod_device_alloc(SimlodContext* ctx, uint64_t bytes, uint64_t* out) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CUdeviceptr p = 0;
    CU(D(cuMemAlloc)(&p, (size_t)bytes));
    *out = (uint64_t)p;
    return SIMLOD_OK;
}
int simlod_device_free(SimlodContext* ctx, uint64_t ptr) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CU(D(cuMemFree)((CUdeviceptr)ptr));
    return SIMLOD_OK;
}

int simlod_get_launch_info(SimlodContext* ctx, uint64_t* launches, uint32_t* construct_blocks, uint32_t* render_blocks, uint32_t* num_sms) {
    if (!ctx) return fail(SIMLOD_ERR_INVALID, "null context");
    if (launches) *launches = ctx->launches;
    if (construct_blocks) *construct_blocks = ctx->constructBlocks;
    if (render_blocks) *render_blocks = ctx->renderBlocks;
    if (num_sms) *num_sms = (uint32_t)ctx->numSMs;
    return SIMLOD_OK;
}

int simlod_get_numa_node(SimlodContext* ctx, int* node) {
    if (!ctx || !node) return fail(SIMLOD_ERR_INVALID, "null argument");
    *node = ctx->numaNode;
    return SIMLOD_OK;
}

int simlod_device_rcp(SimlodContext* ctx, float x, float* out) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CUdeviceptr dst = ctx->scratch4;
    void* args[] = {&x, &dst};
    CU(D(cuLaunchKernel)(ctx->fnRcp, 1, 1, 1, 1, 1, 1, 0, ctx->streamMain, args, nullptr));
    ctx->launches++;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    CU(D(cuMemcpyDtoH)(out, dst, 4));
    return SIMLOD_OK;
}

int simlod_generate(SimlodContext* ctx, int kind, uint64_t n_total, uint64_t first, uint64_t count, uint64_t seed, float size, uint64_t device_points) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!device_points && count) return fail(SIMLOD_ERR_INVALID, "null destination");
    if (first + count > n_total && kind != SIMLOD_GEN_UNIFORM) return fail(SIMLOD_ERR_INVALID, "range [%llu, %llu) outside the %llu-point stream", (unsigned long long)first, (unsigned long long)(first + count), (unsigned long long)n_total);
    if (count == 0) return SIMLOD_OK;
    CUdeviceptr dst = (CUdeviceptr)device_points;
    unsigned blocks = (unsigned)std::min<uint64_t>((count + 255) / 256, (uint64_t)ctx->numSMs * 16);
    if (kind == SIMLOD_GEN_UNIFORM) {
        void* args[] = {&dst, &first, &count, &seed, &size};
        CU(D(cuLaunchKernel)(ctx->fnGenUniform, blocks, 1, 1, 256, 1, 1, 0, ctx->streamMain, args, nullptr));
    } else if (kind == SIMLOD_GEN_TERRAIN || kind == SIMLOD_GEN_SHELL) {
        void* args[] = {&dst, &n_total, &first, &count, &seed};
        CU(D(cuLaunchKernel)(kind == SIMLOD_GEN_TERRAIN ? ctx->fnGenTerrain : ctx->fnGenShell, blocks, 1, 1, 256, 1, 1, 0, ctx->streamMain, args, nullptr));
    } else {
        return fail(SIMLOD_ERR_INVALID, "unknown generator %d", kind);
    }
    ctx->launches++;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    return SIMLOD_OK;
}

int simlod_synchronize(SimlodContext* ctx) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CU(D(cuStreamSynchronize)(ctx->streamUpload));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    return SIMLOD_OK;
}

int simlod_flush_l2(SimlodContext* ctx) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CUdeviceptr dst = ctx->flushBuf;
    uint64_t count = L2_FLUSH_BYTES / 16;
    uint32_t value = 0;
    void* args[] = {&dst, &count, &value};
    CU(D(cuLaunchKernel)(ctx->fnFill, (unsigned)(ctx->numSMs * 8), 1, 1, 256, 1, 1, 0, ctx->streamMain, args, nullptr));
    ctx->launches++;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    return SIMLOD_OK;
}

// ---- spatial exchange (SURVEY.md §8f-3); kernels in partition.cu ----------------------------------------
namespace {
constexpr uint32_t PART_MAX_RANKS = 8, PART_MAX_CELLS = 512, PART_BLOCK = 256, PART_SLOTS = 64;
struct PartitionParams {             // mirrors partition.cu
    float minx, miny, minz, size;
    uint32_t level, numRanks, count, perBlock;
    uint8_t owner[PART_MAX_CELLS];
};
struct ScatterTargets { uint64_t ptr[PART_MAX_RANKS]; uint64_t offset[PART_MAX_RANKS]; uint64_t signal[PART_MAX_RANKS]; uint32_t signalValue, pad; };

// per counted batch: blockHist[blocks][8] | blockBase[blocks][8] | totals[8] | cellCounts[512]
uint64_t partSlotBytes(uint32_t blocks) { return (uint64_t)blocks * PART_MAX_RANKS * 4 * 2 + PART_MAX_RANKS * 4 + PART_MAX_CELLS * 4; }
// scratch tail after the slots: blocksDone (scatter) | timedOut | blocksDone (composite) | pad
int partScratchEnsure(SimlodContext* ctx) {
    if (ctx->partScratch) return SIMLOD_OK;
    const size_t bytes = (size_t)(partSlotBytes((uint32_t)ctx->numSMs * 4) * PART_SLOTS + 16);
    CU(D(cuMemAlloc)(&ctx->partScratch, bytes));
    CU(D(cuMemsetD8)(ctx->partScratch, 0, bytes));
    return SIMLOD_OK;
}

int partitionSetup(SimlodContext* ctx, uint32_t count, const SimlodPartitionPlan* plan, PartitionParams* p, uint32_t* blocks) {
    if (!plan) return fail(SIMLOD_ERR_INVALID, "null plan");
    if (plan->level < 1 || plan->level > 3) return fail(SIMLOD_ERR_INVALID, "partition level %u outside 1..3", plan->level);
    if (plan->num_ranks < 1 || plan->num_ranks > PART_MAX_RANKS) return fail(SIMLOD_ERR_INVALID, "partition over %u ranks (1..8)", plan->num_ranks);
    const uint32_t numCells = 1u << (3 * plan->level);
    for (uint32_t c = 0; c < numCells; c++)
        if (plan->owner[c] >= plan->num_ranks) return fail(SIMLOD_ERR_INVALID, "cell %u is owned by rank %u of %u", c, plan->owner[c], plan->num_ranks);
    const float sx = ctx->uniforms.boxMax[0] - ctx->uniforms.boxMin[0], sy = ctx->uniforms.boxMax[1] - ctx->uniforms.boxMin[1],
                sz = ctx->uniforms.boxMax[2] - ctx->uniforms.boxMin[2];
    p->minx = ctx->uniforms.boxMin[0]; p->miny = ctx->uniforms.boxMin[1]; p->minz = ctx->uniforms.boxMin[2];
    p->size = std::max(std::max(sx, sy), sz);                                       // voxels.cu:860-863
    p->level = plan->level; p->numRanks = plan->num_ranks; p->count = count;
    *blocks = (uint32_t)ctx->numSMs * 4;
    const uint32_t per = (count + *blocks - 1) / *blocks;
    p->perBlock = std::max(PART_BLOCK, (per + PART_BLOCK - 1) / PART_BLOCK * PART_BLOCK);
    memset(p->owner, 0, sizeof(p->owner));
    memcpy(p->owner, plan->owner, numCells);
    return partScratchEnsure(ctx);
}
}  // namespace

int simlod_partition_count(SimlodContext* ctx, uint64_t device_points, uint32_t count, const SimlodPartitionPlan* plan,
                           uint64_t* rank_counts, uint64_t* cell_counts) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!rank_counts) return fail(SIMLOD_ERR_INVALID, "null argument");
    if (!device_points && count) return fail(SIMLOD_ERR_INVALID, "null points");
    PartitionParams p; uint32_t blocks = 0;
    rc = partitionSetup(ctx, count, plan, &p, &blocks); if (rc) return rc;
    // a batch may be counted well ahead of its scatter (planning a window of steps): its block bases stay in a slot
    uint32_t slot = PART_SLOTS;
    for (uint32_t i = 0; i < PART_SLOTS; i++)
        if (ctx->partSlots[i].valid && ctx->partSlots[i].points == device_points && ctx->partSlots[i].count == count) slot = i;
    if (slot == PART_SLOTS) { slot = ctx->partNextSlot; ctx->partNextSlot = (ctx->partNextSlot + 1) % PART_SLOTS; }
    CUdeviceptr pts = (CUdeviceptr)device_points;
    CUdeviceptr blockHist = ctx->partScratch + partSlotBytes(blocks) * slot, blockBase = blockHist + (size_t)blocks * PART_MAX_RANKS * 4,
                totals = blockBase + (size_t)blocks * PART_MAX_RANKS * 4, cells = totals + PART_MAX_RANKS * 4;
    CU(D(cuMemsetD8Async)(cells, 0, PART_MAX_CELLS * 4, ctx->streamMain));
    { void* args[] = {&p, &pts, &blockHist, &cells};
      CU(D(cuLaunchKernel)(ctx->fnPartCount, blocks, 1, 1, PART_BLOCK, 1, 1, 0, ctx->streamMain, args, nullptr)); }
    { void* args[] = {&blockHist, &blocks, &blockBase, &totals};
      CU(D(cuLaunchKernel)(ctx->fnPartScan, 1, 1, 1, PART_BLOCK, 1, 1, 0, ctx->streamMain, args, nullptr)); }
    ctx->launches += 2;
    uint32_t host[PART_MAX_RANKS + PART_MAX_CELLS];
    CU(D(cuMemcpyDtoHAsync)(host, totals, sizeof(host), ctx->streamMain));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    for (uint32_t d = 0; d < plan->num_ranks; d++) rank_counts[d] = host[d];
    if (cell_counts) for (uint32_t c = 0; c < (1u << (3 * plan->level)); c++) cell_counts[c] = host[PART_MAX_RANKS + c];
    ctx->partSlots[slot].points = device_points; ctx->partSlots[slot].count = count; ctx->partSlots[slot].valid = true;
    return SIMLOD_OK;
}

int simlod_partition_scatter(SimlodContext* ctx, uint64_t device_points, uint32_t count, const SimlodPartitionPlan* plan,
                             const uint64_t* dest_ptrs, const uint64_t* dest_offsets, const uint64_t* signal_ptrs, uint32_t signal_value) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!dest_ptrs || !dest_offsets) return fail(SIMLOD_ERR_INVALID, "null argument");
    uint32_t slot = PART_SLOTS;
    for (uint32_t i = 0; i < PART_SLOTS; i++)
        if (ctx->partSlots[i].valid && ctx->partSlots[i].points == device_points && ctx->partSlots[i].count == count) slot = i;
    if (slot == PART_SLOTS) return fail(SIMLOD_ERR_INVALID, "simlod_partition_scatter must follow simlod_partition_count on the same batch");
    PartitionParams p; uint32_t blocks = 0;
    rc = partitionSetup(ctx, count, plan, &p, &blocks); if (rc) return rc;
    ScatterTargets t;
    memset(&t, 0, sizeof(t));
    for (uint32_t d = 0; d < plan->num_ranks; d++) {
        if (!dest_ptrs[d]) return fail(SIMLOD_ERR_INVALID, "null destination for rank %u", d);
        t.ptr[d] = dest_ptrs[d]; t.offset[d] = dest_offsets[d];
        if (signal_ptrs) {
            if (!signal_ptrs[d]) return fail(SIMLOD_ERR_INVALID, "null signal word for rank %u", d);
            t.signal[d] = signal_ptrs[d];
        }
    }
    t.signalValue = signal_value;
    CUdeviceptr pts = (CUdeviceptr)device_points;
    CUdeviceptr blockBase = ctx->partScratch + partSlotBytes(blocks) * slot + (size_t)blocks * PART_MAX_RANKS * 4;
    CUdeviceptr blocksDone = ctx->partScratch + partSlotBytes(blocks) * PART_SLOTS;
    void* args[] = {&p, &t, &pts, &blockBase, &blocksDone};
    CU(D(cuLaunchKernel)(ctx->fnPartScatter, blocks, 1, 1, PART_BLOCK, 1, 1, 0, ctx->streamMain, args, nullptr));
    ctx->launches++;
    ctx->partSlots[slot].valid = false;
    return SIMLOD_OK;
}

int simlod_partition_wait(SimlodContext* ctx, uint64_t local_flags, uint32_t num_ranks, uint32_t value, uint32_t timeout_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!local_flags || num_ranks < 1 || num_ranks > PART_MAX_RANKS) return fail(SIMLOD_ERR_INVALID, "bad flags / rank count");
    { int rcs = partScratchEnsure(ctx); if (rcs) return rcs; }
    CUdeviceptr flags = (CUdeviceptr)local_flags;
    CUdeviceptr timedOut = ctx->partScratch + partSlotBytes((uint32_t)ctx->numSMs * 4) * PART_SLOTS + 4;
    uint64_t cycles = (uint64_t)(timeout_ms ? timeout_ms : 10000) * 2000000ull;          // SM clock ~2 GHz
    void* args[] = {&flags, &num_ranks, &value, &cycles, &timedOut};
    CU(D(cuLaunchKernel)(ctx->fnPartWait, 1, 1, 1, 32, 1, 1, 0, ctx->streamMain, args, nullptr));
    ctx->launches++;
    uint32_t host = 0;
    CU(D(cuMemcpyDtoHAsync)(&host, timedOut, 4, ctx->streamMain));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    if (host) {
        CU(D(cuMemsetD8)(timedOut, 0, 4));
        return fail(SIMLOD_ERR_CUDA, "spatial exchange: rank %u did not signal step %u within %u ms", host - 1, value, timeout_ms ? timeout_ms : 10000);
    }
    return SIMLOD_OK;
}

// ---- depth compositing of the ranks' framebuffers over peer memory (DESIGN.md §9.3) ------------------------
namespace {
struct CompositeArgs { uint64_t fb[PART_MAX_RANKS]; uint64_t signal[PART_MAX_RANKS]; uint64_t numWords; uint32_t numRanks, rank, signalValue, pad; };
struct SignalArgs { uint64_t signal[PART_MAX_RANKS]; uint32_t numRanks, value; };
}  // namespace

int simlod_export_framebuffer(SimlodContext* ctx, uint64_t dst_device) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!dst_device) return fail(SIMLOD_ERR_INVALID, "null destination");
    CU(D(cuMemcpyDtoDAsync)((CUdeviceptr)dst_device, ctx->buf.renderbuffer + FB_OFFSET, (size_t)ctx->cfg.width * ctx->cfg.height * 8, ctx->streamMain));
    return SIMLOD_OK;
}

int simlod_peer_signal(SimlodContext* ctx, const uint64_t* signal_ptrs, uint32_t num_ranks, uint32_t value) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!signal_ptrs || num_ranks < 1 || num_ranks > PART_MAX_RANKS) return fail(SIMLOD_ERR_INVALID, "bad signal words / rank count");
    SignalArgs a;
    memset(&a, 0, sizeof(a));
    for (uint32_t d = 0; d < num_ranks; d++) { if (!signal_ptrs[d]) return fail(SIMLOD_ERR_INVALID, "null signal word for rank %u", d); a.signal[d] = signal_ptrs[d]; }
    a.numRanks = num_ranks; a.value = value;
    void* args[] = {&a};
    CU(D(cuLaunchKernel)(ctx->fnPeerSignal, 1, 1, 1, 32, 1, 1, 0, ctx->streamMain, args, nullptr));
    ctx->launches++;
    return SIMLOD_OK;
}

int simlod_composite_framebuffers(SimlodContext* ctx, const uint64_t* fb_ptrs, uint32_t num_ranks, uint32_t rank,
                                  const uint64_t* signal_ptrs, uint32_t signal_value) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!fb_ptrs || num_ranks < 1 || num_ranks > PART_MAX_RANKS || rank >= num_ranks) return fail(SIMLOD_ERR_INVALID, "bad framebuffer list / rank");
    rc = partScratchEnsure(ctx); if (rc) return rc;
    CompositeArgs a;
    memset(&a, 0, sizeof(a));
    for (uint32_t d = 0; d < num_ranks; d++) {
        if (!fb_ptrs[d]) return fail(SIMLOD_ERR_INVALID, "null framebuffer for rank %u", d);
        a.fb[d] = fb_ptrs[d];
        if (signal_ptrs) { if (!signal_ptrs[d]) return fail(SIMLOD_ERR_INVALID, "null signal word for rank %u", d); a.signal[d] = signal_ptrs[d]; }
    }
    a.numWords = (uint64_t)ctx->cfg.width * ctx->cfg.height;
    a.numRanks = num_ranks; a.rank = rank; a.signalValue = signal_value;
    CUdeviceptr blocksDone = ctx->partScratch + partSlotBytes((uint32_t)ctx->numSMs * 4) * PART_SLOTS + 8;
    void* args[] = {&a, &blocksDone};
    CU(D(cuLaunchKernel)(ctx->fnComposite, (unsigned)ctx->numSMs * 4, 1, 1, PART_BLOCK, 1, 1, 0, ctx->streamMain, args, nullptr));
    ctx->launches++;
    return SIMLOD_OK;
}

}  // extern "C"
