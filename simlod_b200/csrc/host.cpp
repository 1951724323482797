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
#include <sys/stat.h>
#include <sys/syscall.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <limits>
#include <mutex>
#include <thread>
#include <cstdarg>
#include <cstdio>
#include <cctype>
#include <cstring>
#include <fstream>
#include <cmath>
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
extern const unsigned char simlod_cubin_export[];
extern const unsigned char simlod_cubin_import[];
extern const unsigned char simlod_cubin_query[];
extern const unsigned char simlod_cubin_pick[];
extern const unsigned char simlod_cubin_nearest[];
extern const unsigned char simlod_cubin_ray[];
extern const unsigned char simlod_cubin_radius[];
extern const unsigned char simlod_cubin_las_write[];
extern const unsigned char simlod_cubin_heightmap[];
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
constexpr uint64_t L2_FLUSH_BYTES = 512ull << 20;

struct Program {
    CUmodule module = nullptr;
    CUfunction fn = nullptr;
    CUfunction fnClip = nullptr;       // the render program's simlod_render_clip; null in a module without it
    bool builtin = true;
};

// The embedded images of the kernels that are launched outside the three swappable programs, and those kernels: one
// row each, {enum value, image, kernel name}. createResources loads every image and looks up every kernel.
enum Image { IMG_UTIL, IMG_LAS, IMG_GEN, IMG_PARTITION, IMG_EXPORT, IMG_QUERY, IMG_IMPORT, IMG_PICK, IMG_NEAREST, IMG_RAY, IMG_RADIUS, IMG_LAS_WRITE, IMG_HEIGHTMAP, NUM_IMAGES };
const unsigned char* const IMAGES[NUM_IMAGES] = {simlod_cubin_util, simlod_cubin_las, simlod_cubin_gen, simlod_cubin_partition,
                                                 simlod_cubin_export, simlod_cubin_query, simlod_cubin_import, simlod_cubin_pick,
                                                 simlod_cubin_nearest, simlod_cubin_ray, simlod_cubin_radius, simlod_cubin_las_write,
                                                 simlod_cubin_heightmap};
#define KERNEL_LIST(X)                                                                                    \
    X(K_RCP, IMG_UTIL, "simlod_util_rcp") X(K_FILL, IMG_UTIL, "simlod_util_fill")                         \
    X(K_LAS, IMG_LAS, "simlod_las_decode")                                                                \
    X(K_GEN_UNIFORM, IMG_GEN, "simlod_gen_uniform") X(K_GEN_TERRAIN, IMG_GEN, "simlod_gen_terrain")       \
    X(K_GEN_SHELL, IMG_GEN, "simlod_gen_shell")                                                           \
    X(K_PART_COUNT, IMG_PARTITION, "simlod_partition_count") X(K_PART_SCAN, IMG_PARTITION, "simlod_partition_scan") \
    X(K_PART_SCATTER, IMG_PARTITION, "simlod_partition_scatter") X(K_PART_WAIT, IMG_PARTITION, "simlod_partition_wait") \
    X(K_COMPOSITE, IMG_PARTITION, "simlod_composite_min") X(K_PEER_SIGNAL, IMG_PARTITION, "simlod_peer_signal") \
    X(K_EXPORT_PLAN, IMG_EXPORT, "simlod_export_plan") X(K_EXPORT_PLAN_VIEW, IMG_EXPORT, "simlod_export_plan_view") \
    X(K_EXPORT_VIEW_FLAGS, IMG_EXPORT, "simlod_export_view_flags") X(K_EXPORT_COLLECT, IMG_EXPORT, "simlod_export_collect") \
    X(K_EXPORT_GATHER, IMG_EXPORT, "simlod_export_gather") X(K_EXPORT_GATHER_WINDOW, IMG_EXPORT, "simlod_export_gather_window") \
    X(K_EXPORT_COUNTERS, IMG_EXPORT, "simlod_export_counters")                                            \
    X(K_QUERY_PLAN, IMG_QUERY, "simlod_query_plan") X(K_QUERY_COUNT, IMG_QUERY, "simlod_query_count")     \
    X(K_QUERY_SCAN, IMG_QUERY, "simlod_query_scan") X(K_QUERY_WRITE, IMG_QUERY, "simlod_query_write")     \
    X(K_IMPORT_NODES, IMG_IMPORT, "simlod_import_nodes") X(K_IMPORT_LINK, IMG_IMPORT, "simlod_import_link") \
    X(K_IMPORT_CLEAR_GRIDS, IMG_IMPORT, "simlod_import_clear_grids") X(K_IMPORT_SCATTER, IMG_IMPORT, "simlod_import_scatter") \
    X(K_IMPORT_VOXELS, IMG_IMPORT, "simlod_import_voxels") X(K_IMPORT_COUNT_GRIDS, IMG_IMPORT, "simlod_import_count_grids") \
    X(K_PICK_CLEAR, IMG_PICK, "simlod_pick_clear") X(K_PICK_KEY, IMG_PICK, "simlod_pick_key")             \
    X(K_PICK_INDEX, IMG_PICK, "simlod_pick_index") X(K_PICK_WRITE, IMG_PICK, "simlod_pick_write")             \
    X(K_NEAREST_LOCATE, IMG_NEAREST, "simlod_nearest_locate") X(K_NEAREST_SCAN, IMG_NEAREST, "simlod_nearest_scan") \
    X(K_NEAREST_SCATTER, IMG_NEAREST, "simlod_nearest_scatter") X(K_NEAREST_SEARCH, IMG_NEAREST, "simlod_nearest_search") \
    X(K_RAY_CHECK, IMG_RAY, "simlod_ray_check") X(K_RAY_TRACE, IMG_RAY, "simlod_ray_trace")                 \
    X(K_RADIUS_COUNT, IMG_RADIUS, "simlod_radius_count") X(K_RADIUS_REDUCE, IMG_RADIUS, "simlod_radius_reduce") \
    X(K_RADIUS_SCAN, IMG_RADIUS, "simlod_radius_scan") X(K_RADIUS_WRITE, IMG_RADIUS, "simlod_radius_write") \
    X(K_LAS_ENCODE, IMG_LAS_WRITE, "simlod_las_encode")                                                   \
    X(K_HEIGHTMAP_ACCUMULATE, IMG_HEIGHTMAP, "simlod_heightmap_accumulate")                               \
    X(K_HEIGHTMAP_FINALIZE, IMG_HEIGHTMAP, "simlod_heightmap_finalize")
#define X(k, image, name) k,
enum Kernel { KERNEL_LIST(X) NUM_KERNELS };
#undef X
struct KernelRow { Image image; const char* name; };
#define X(k, image, name) {image, name},
const KernelRow KERNELS[NUM_KERNELS] = {KERNEL_LIST(X)};
#undef X

}  // namespace

#include "loader_pool.h"
#include "construct_layout.cuh"
#include "kernel_args.h"
#include "render_layout.cuh"

struct SimlodContext {
    CUdevice device = 0;
    CUcontext primary = nullptr;
    int numSMs = 0;
    CUstream streamMain = nullptr, streamUpload = nullptr;
    CUevent evStart = nullptr, evEnd = nullptr, evTotalStart = nullptr, evTotalEnd = nullptr;
    CUevent evSlot[RING_SLOTS] = {};    // recorded on the upload stream when the batch in that ring slot has been published
    SimlodConfig cfg{};
    SimlodUniforms uniforms{};
    SimlodBuffers buf{};
    CUdeviceptr numBatchesUploaded = 0, batchSizes = 0, frameStart = 0, cudaprint = 0, scratch4 = 0, flushBuf = 0;
    CUarray colorArray = nullptr;
    CUsurfObject surface = 0;
    SimlodStats* hStats = nullptr;     // pinned
    // kernel_construct launches enqueued back to back on streamMain, each followed by an asynchronous copy of Stats
    // (enqueueLaunch / retireLaunch)
    struct LaunchQueue {
        static constexpr uint32_t DEPTH = 8;
        CUevent ev[DEPTH][2] = {};     // start / end of the launch in slot k
        CUevent statsDone[DEPTH] = {}; // the Stats snapshot behind slot k has landed
        SimlodStats* snap = nullptr;   // pinned, one snapshot per slot
        uint32_t want[DEPTH] = {};     // the launch in slot k started once batches [0, want) were published
        uint32_t head = 0, size = 0;   // oldest slot in flight, launches in flight
        uint32_t stalled = 0;          // snapshots in a row in which published batches waited and none was consumed
        float kernelMs = 0.0f;         // summed time of the retired launches
    } queue;
    struct PublishMirror { uint32_t sizes[RING_SLOTS]; uint32_t count; uint32_t pad[13]; };   // 256 B
    PublishMirror* hPublish = nullptr; // pinned, 16 snapshots of {batchSizes[50], numBatchesUploaded} for grouped publication
    CUevent evPublish[16] = {};        // the copies out of mirror i have completed
    uint32_t hostSizes[RING_SLOTS] = {};   // what batchSizes[] holds on the device once everything enqueued has run
    uint32_t unpublished = 0;          // batches copied into the ring but not yet published (sizes + counter)
    uint32_t publishIndex = 0;
    Program programs[3];
    CUmodule modules[NUM_IMAGES] = {};
    CUfunction fn[NUM_KERNELS] = {};
    CUdeviceptr partScratch = 0;       // spatial exchange: PART_SLOTS x (blockHist | blockBase | totals | cellCounts), then blocksDone, timedOut
    struct PartSlot { uint64_t points = 0; uint32_t count = 0; bool valid = false; } partSlots[64];   // counted batches awaiting their scatter
    uint32_t partNextSlot = 0;
    // raw LAS records from host memory: stagingSlots slots of stagingSlotBytes, filled on streamCopy and decoded on
    // streamUpload; a copy waits for evStagingFree of its slot (the last decode out of it), a decode for evStaged
    static constexpr uint32_t MAX_STAGING_SLOTS = 16;
    CUstream streamCopy = nullptr;
    CUdeviceptr staging = 0;
    uint64_t stagingSlotBytes = 0;
    uint32_t stagingSlots = 0, stagingNext = 0;
    CUevent evStaged[MAX_STAGING_SLOTS] = {}, evStagingFree[MAX_STAGING_SLOTS] = {};
    CUdeviceptr exportScratch = 0;     // octree export and region query: see scratchFor()
    uint64_t exportScratchBytes = 0;
    void* hExportCtl = nullptr;        // pinned copy of the control structs read back (StageClock::finish)
    CUdeviceptr queryScratch = 0;      // the plan's consumers, one at a time: pick's frames, the buckets and passes of k
    uint64_t queryScratchBytes = 0;    // nearest and radius, RayCtl, the height map's accumulators
    CUdeviceptr fileWindow = 0;        // octree files: FILE_WINDOW_BYTES of samples staged on the device
    CUdeviceptr fileTables = 0;        // octree load: records | plan | error word, sized for nodes[]
    CUdeviceptr lasWindow = 0;         // LAS writer: one window of records, then LasWriteCtl
    CUevent evLas[2][4] = {};          // LAS writer, per pool half: encode start, encode end, copy start, records copied out
    uint64_t fileTablesBytes = 0;
    void* pinnedPool = nullptr;        // POOL_BYTES page-locked: the file streamer's slots, one batch of records each
    LoaderPool* loaderPool = nullptr;
    CUevent evPool[32] = {};           // H2D copy out of pool slot i has been enqueued and completed
    uint32_t uploaded = 0;             // batches published to the device
    uint32_t processed = 0;            // Stats::batchletIndex as last read
    uint64_t launches = 0;
    uint32_t constructBlocks = 0, renderBlocks = 0;
    int numaNode = -1;                 // host NUMA node the page-locked buffers were placed on (-1: unknown)
    uint64_t frameCounter = 0;
    SimlodClip clip{};                 // simlod_set_clip; mode SIMLOD_CLIP_NONE: none
};

namespace {

int devAlloc(uint64_t* out, uint64_t bytes) {
    CUdeviceptr p = 0;
    CU(D(cuMemAlloc)(&p, (size_t)bytes));
    *out = (uint64_t)p;
    return SIMLOD_OK;
}
#define ALLOC(field, bytes) do { int _rc = devAlloc(&(field), (bytes)); if (_rc) return _rc; } while (0)

// a device allocation of at least `bytes`, replaced by a larger one (its contents dropped) when it is smaller
int growDevice(CUdeviceptr* p, uint64_t* have, uint64_t bytes) {
    if (*have >= bytes) return SIMLOD_OK;
    if (*p) CU(D(cuMemFree)(*p));
    *p = 0;
    *have = 0;
    CU(D(cuMemAlloc)(p, bytes));
    *have = bytes;
    return SIMLOD_OK;
}

// a device address as the typed pointer a kernel argument struct holds
struct DevPtr {
    CUdeviceptr p;
    template <class T> operator T*() const { return reinterpret_cast<T*>((uintptr_t)p); }
};
DevPtr devPtr(CUdeviceptr p) { return DevPtr{p}; }

// Every kernel launch of the library, counted in ctx->launches once the driver has accepted it. The arguments bind by
// lvalue reference, so each reaches the kernel with the type it is declared with: a temporary (cap + 1) does not bind.
int launchParams(SimlodContext* ctx, bool cooperative, CUfunction fn, unsigned grid, unsigned block, CUstream s, void** params) {
    if (cooperative) CU(D(cuLaunchCooperativeKernel)(fn, grid, 1, 1, block, 1, 1, 0, s, params));
    else CU(D(cuLaunchKernel)(fn, grid, 1, 1, block, 1, 1, 0, s, params, nullptr));
    ctx->launches++;
    return SIMLOD_OK;
}
template <class... A>
int launch(SimlodContext* ctx, CUfunction fn, unsigned grid, unsigned block, CUstream s, A&... args) {
    void* params[] = {(void*)&args...};
    return launchParams(ctx, false, fn, grid, block, s, params);
}
template <class... A>
int launchCooperative(SimlodContext* ctx, CUfunction fn, unsigned grid, unsigned block, CUstream s, A&... args) {
    void* params[] = {(void*)&args...};
    return launchParams(ctx, true, fn, grid, block, s, params);
}

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
    // the clipped frame runs on kernel_render's grid (the EDL tile coverage depends on it), so it must be resident there
    if (CUfunction clip = ctx->programs[SIMLOD_PROGRAM_RENDER].fnClip) {
        int occClip = 0;
        CU(D(cuOccupancyMaxActiveBlocksPerMultiprocessor)(&occClip, clip, 256, 0));
        if (occClip < per) return fail(SIMLOD_ERR_MODULE, "simlod_render_clip is resident with %d blocks per SM, kernel_render's grid needs %d", occClip, per);
    }
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
    CUfunction fnClip = nullptr;       // optional: a render module without it renders, but not with a clip set
    if (program == SIMLOD_PROGRAM_RENDER && D(cuModuleGetFunction)(&fnClip, mod, "simlod_render_clip") != CUDA_SUCCESS) fnClip = nullptr;
    Program& p = ctx->programs[program];
    if (p.module) D(cuModuleUnload)(p.module);
    p.module = mod; p.fn = fn; p.fnClip = fnClip; p.builtin = builtin;
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

// enqueue one kernel_construct launch between the events `start` and `end` without waiting for it. `points` replaces the
// ring as the kernel's points argument (the zero-copy window of simlod_insert_device); 0 keeps the ring.
int launchConstruct(SimlodContext* ctx, CUevent start, CUevent end, CUdeviceptr points = 0) {
    SimlodUniforms u = ctx->uniforms;
    u.frameCounter = ctx->frameCounter;
    CUdeviceptr ring = points ? points : ctx->buf.ring, momentary = ctx->buf.momentary, persistent = ctx->buf.persistent, nodes = ctx->buf.nodes,
                stats = ctx->buf.stats, frameStart = ctx->frameStart, cudaprint = ctx->cudaprint,
                nbu = ctx->numBatchesUploaded, bs = ctx->batchSizes;
    CU(D(cuEventRecord)(start, ctx->streamMain));
    int rc = launchCooperative(ctx, ctx->programs[SIMLOD_PROGRAM_CONSTRUCT].fn, ctx->constructBlocks, 256, ctx->streamMain,
                               u, ring, momentary, persistent, nodes, stats, frameStart, cudaprint, nbu, bs);   // main.cpp:374-382
    if (rc) return rc;
    CU(D(cuEventRecord)(end, ctx->streamMain));
    return SIMLOD_OK;
}

// Launch queue: a launch waits on the upload stream until batches [0, want) are published (the slot event of batch
// want - 1), and an asynchronous copy of Stats follows it, as the reference copies Stats every frame (main.cpp:1201-1216).
// The host learns what the device has consumed from these snapshots, so it never drains the launch stream to decide what
// to do next and the GPU does not idle between launches.
int enqueueLaunch(SimlodContext* ctx, uint32_t want, CUdeviceptr points) {
    SimlodContext::LaunchQueue& q = ctx->queue;
    const uint32_t k = (q.head + q.size) % q.DEPTH;
    CU(D(cuStreamWaitEvent)(ctx->streamMain, ctx->evSlot[(want - 1u) % RING_SLOTS], 0));
    int rc = launchConstruct(ctx, q.ev[k][0], q.ev[k][1], points); if (rc) return rc;
    CU(D(cuMemcpyDtoHAsync)(&q.snap[k], ctx->buf.stats, sizeof(SimlodStats), ctx->streamMain));
    CU(D(cuEventRecord)(q.statsDone[k], ctx->streamMain));
    q.want[k] = want;
    q.size++;
    return SIMLOD_OK;
}

// Take in the snapshot of the oldest launch in flight, waiting for it if `block`: 1 if one was taken in, 0 if none is
// ready, < 0 on error. The snapshot becomes hStats / processed and is checked: a full heap, dropped samples, and more
// than 4 launches in a row that found published batches and consumed none, with nothing left in flight.
int retireLaunch(SimlodContext* ctx, bool block) {
    SimlodContext::LaunchQueue& q = ctx->queue;
    if (q.size == 0) return 0;
    const uint32_t k = q.head;
    if (!block) {
        CUresult r = D(cuEventQuery)(q.statsDone[k]);
        if (r == CUDA_ERROR_NOT_READY) return 0;
        if (r != CUDA_SUCCESS) return fail(SIMLOD_ERR_CUDA, "event query failed (%d)", (int)r);
    } else {
        CUresult r = D(cuEventSynchronize)(q.statsDone[k]);
        if (r != CUDA_SUCCESS) { const char* e = nullptr; D(cuGetErrorString)(r, &e); return fail(SIMLOD_ERR_CUDA, "kernel_construct failed: %s (%d)", e ? e : "?", (int)r); }
    }
    float ms = 0.0f;
    D(cuEventElapsedTime)(&ms, q.ev[k][0], q.ev[k][1]);
    q.kernelMs += ms;
    const uint32_t before = ctx->processed;
    *ctx->hStats = q.snap[k];
    ctx->processed = ctx->hStats->batchletIndex;
    q.head = (q.head + 1) % q.DEPTH;
    q.size--;
    q.stalled = ctx->processed == before && before < q.want[k] ? q.stalled + 1 : 0;
    if (ctx->hStats->memCapacityReached) return fail(SIMLOD_ERR_CAPACITY, "persistent heap almost full after %llu points", (unsigned long long)ctx->hStats->numPointsProcessed);
    int rc = checkOverflow(ctx); if (rc) return rc;
    if (q.size == 0 && q.stalled > 4) return fail(SIMLOD_ERR_CUDA, "kernel_construct makes no progress (%u of %u batches consumed)", ctx->processed, ctx->uploaded);
    return 1;
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
    CU(D(cuStreamCreate)(&ctx->streamCopy, CU_STREAM_NON_BLOCKING));
    for (uint32_t i = 0; i < ctx->MAX_STAGING_SLOTS; i++) {
        CU(D(cuEventCreate)(&ctx->evStaged[i], CU_EVENT_DISABLE_TIMING));
        CU(D(cuEventCreate)(&ctx->evStagingFree[i], CU_EVENT_DISABLE_TIMING));
    }
    CU(D(cuEventCreate)(&ctx->evStart, CU_EVENT_DEFAULT));
    CU(D(cuEventCreate)(&ctx->evEnd, CU_EVENT_DEFAULT));
    CU(D(cuEventCreate)(&ctx->evTotalStart, CU_EVENT_DEFAULT));
    CU(D(cuEventCreate)(&ctx->evTotalEnd, CU_EVENT_DEFAULT));
    for (auto& pair : ctx->queue.ev) for (CUevent& e : pair) CU(D(cuEventCreate)(&e, CU_EVENT_DEFAULT));
    for (uint64_t i = 0; i < RING_SLOTS; i++) CU(D(cuEventCreate)(&ctx->evSlot[i], CU_EVENT_DISABLE_TIMING));

    // programs (main.cpp:603-626)
    for (int p = 0; p < 3; p++) {
        int rc = loadProgram(ctx, p, builtinImage(p), true);
        if (rc != SIMLOD_OK) return rc;
    }
    for (int i = 0; i < NUM_IMAGES; i++) CU(D(cuModuleLoadData)(&ctx->modules[i], IMAGES[i]));
    for (int k = 0; k < NUM_KERNELS; k++) CU(D(cuModuleGetFunction)(&ctx->fn[k], ctx->modules[KERNELS[k].image], KERNELS[k].name));

    // buffers (main.cpp:552-586)
    SimlodBuffers& b = ctx->buf;
    b.momentary_bytes = config->momentary_bytes ? config->momentary_bytes : 300000000ull;
    b.nodes_bytes = config->nodes_bytes ? config->nodes_bytes : 40000000ull;
    b.renderbuffer_bytes = config->renderbuffer_bytes ? config->renderbuffer_bytes : 200000000ull;
    b.ring_bytes = RING_SLOTS * SLOT_POINTS * sizeof(SimlodPoint);
    if (rbuf::targetsEnd((uint64_t)config->width * config->height) > b.renderbuffer_bytes) return fail(SIMLOD_ERR_INVALID, "render buffer too small for %ux%u", config->width, config->height);
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
    CU(D(cuMemHostAlloc)((void**)&ctx->queue.snap, ctx->queue.DEPTH * sizeof(SimlodStats), 0));
    CU(D(cuMemHostAlloc)((void**)&ctx->hPublish, 16 * sizeof(SimlodContext::PublishMirror), 0));
    for (int i = 0; i < 16; i++) CU(D(cuEventCreate)(&ctx->evPublish[i], CU_EVENT_DISABLE_TIMING));
    for (CUevent& e : ctx->queue.statsDone) CU(D(cuEventCreate)(&e, CU_EVENT_DISABLE_TIMING));
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
        if (ctx->queue.snap) D(cuMemFreeHost)(ctx->queue.snap);
        if (ctx->hPublish) D(cuMemFreeHost)(ctx->hPublish);
        for (int i = 0; i < 16; i++) if (ctx->evPublish[i]) D(cuEventDestroy)(ctx->evPublish[i]);
        for (CUevent e : ctx->queue.statsDone) if (e) D(cuEventDestroy)(e);
        for (int p = 0; p < 3; p++) if (ctx->programs[p].module) D(cuModuleUnload)(ctx->programs[p].module);
        for (CUmodule m : ctx->modules) if (m) D(cuModuleUnload)(m);
        if (ctx->partScratch) D(cuMemFree)(ctx->partScratch);
        if (ctx->staging) D(cuMemFree)(ctx->staging);
        for (uint32_t i = 0; i < ctx->MAX_STAGING_SLOTS; i++) {
            if (ctx->evStaged[i]) D(cuEventDestroy)(ctx->evStaged[i]);
            if (ctx->evStagingFree[i]) D(cuEventDestroy)(ctx->evStagingFree[i]);
        }
        if (ctx->exportScratch) D(cuMemFree)(ctx->exportScratch);
        if (ctx->hExportCtl) D(cuMemFreeHost)(ctx->hExportCtl);
        if (ctx->queryScratch) D(cuMemFree)(ctx->queryScratch);
        if (ctx->fileWindow) D(cuMemFree)(ctx->fileWindow);
        if (ctx->fileTables) D(cuMemFree)(ctx->fileTables);
        if (ctx->lasWindow) D(cuMemFree)(ctx->lasWindow);
        for (auto& half : ctx->evLas) for (CUevent e : half) if (e) D(cuEventDestroy)(e);
        delete ctx->loaderPool;          // joins the loader threads
        if (ctx->pinnedPool) D(cuMemFreeHost)(ctx->pinnedPool);
        for (int i = 0; i < 32; i++) if (ctx->evPool[i]) D(cuEventDestroy)(ctx->evPool[i]);
        if (ctx->evStart) D(cuEventDestroy)(ctx->evStart);
        if (ctx->evEnd) D(cuEventDestroy)(ctx->evEnd);
        if (ctx->evTotalStart) D(cuEventDestroy)(ctx->evTotalStart);
        if (ctx->evTotalEnd) D(cuEventDestroy)(ctx->evTotalEnd);
        for (auto& pair : ctx->queue.ev) for (CUevent e : pair) if (e) D(cuEventDestroy)(e);
        for (uint64_t i = 0; i < RING_SLOTS; i++) if (ctx->evSlot[i]) D(cuEventDestroy)(ctx->evSlot[i]);
        if (ctx->streamMain) D(cuStreamDestroy)(ctx->streamMain);
        if (ctx->streamUpload) D(cuStreamDestroy)(ctx->streamUpload);
        if (ctx->streamCopy) D(cuStreamDestroy)(ctx->streamCopy);
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
    CU(D(cuStreamSynchronize)(ctx->streamCopy));
    CU(D(cuStreamSynchronize)(ctx->streamUpload));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    CU(D(cuMemsetD8Async)(ctx->buf.nodes, 0, ctx->buf.nodes_bytes, ctx->streamMain));
    SimlodUniforms u = ctx->uniforms;
    u.frameCounter = ctx->frameCounter;
    CUdeviceptr persistent = ctx->buf.persistent, nodes = ctx->buf.nodes, stats = ctx->buf.stats, cudaprint = ctx->cudaprint,
                nbu = ctx->numBatchesUploaded, bs = ctx->batchSizes;
    rc = launchCooperative(ctx, ctx->programs[SIMLOD_PROGRAM_RESET].fn, blocks, threads, ctx->streamMain,
                           u, persistent, nodes, stats, cudaprint, nbu, bs);      // main.cpp:337-345
    if (rc) return rc;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    ctx->uploaded = 0;
    ctx->processed = 0;
    ctx->unpublished = 0;
    memset(ctx->hostSizes, 0, sizeof(ctx->hostSizes));
    return SIMLOD_OK;
}

// the ring slot of the next batch of `count` points and its device address; with back-pressure as main.cpp:1012
static int claimSlot(SimlodContext* ctx, uint32_t count, uint32_t* slot, CUdeviceptr* dst) {
    if (count > SLOT_POINTS) return fail(SIMLOD_ERR_INVALID, "batch of %u points exceeds the ring slot size of %llu", count, (unsigned long long)SLOT_POINTS);
    if (ctx->uploaded - ctx->processed >= RING_SLOTS) {
        int rc = readStats(ctx); if (rc) return rc;
        if (ctx->uploaded - ctx->processed >= RING_SLOTS) return fail(SIMLOD_ERR_RING_FULL, "all %llu ring slots hold unprocessed batches", (unsigned long long)RING_SLOTS);
    }
    *slot = ctx->uploaded % RING_SLOTS;
    *dst = ctx->buf.ring + (uint64_t)*slot * SLOT_POINTS * sizeof(SimlodPoint);
    return SIMLOD_OK;
}

static int uploadCommon(SimlodContext* ctx, const void* host, CUdeviceptr dev, uint32_t count, bool publish = true) {
    int rc = setCurrent(ctx); if (rc) return rc;
    uint32_t slot = 0;
    CUdeviceptr dst = 0;
    rc = claimSlot(ctx, count, &slot, &dst); if (rc) return rc;
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

// The records the decoder accepts and the RGB offset of their format (LasLoader.cpp:179-188): 2 -> 20, 3 / 5 -> 28,
// 7 -> 30, any other format has no colour. The one place these rules live: the batch upload and the file front end
// both ask here.
static int lasRgbOffset(uint32_t format, uint32_t bytesPerPoint, uint32_t* offsetRgb, const char* what = "") {
    if (bytesPerPoint < 12 || bytesPerPoint > 96) return fail(SIMLOD_ERR_INVALID, "%s%sunsupported LAS record size %u", what, *what ? ": " : "", bytesPerPoint);
    uint32_t o = 0;
    if (format == 2) o = 20; else if (format == 3) o = 28;
    if (format == 5) o = 28;
    if (format == 7) o = 30;
    if (o && o + 6 > bytesPerPoint) return fail(SIMLOD_ERR_INVALID, "%s%sLAS format %u does not fit %u-byte records", what, *what ? ": " : "", format, bytesPerPoint);
    *offsetRgb = o;
    return SIMLOD_OK;
}

// device staging slots of at least `bytes` each: as many as fit into 512 MB, between 2 and MAX_STAGING_SLOTS; grown
// (after the streams that use them have drained) when a larger record size needs it
static int ensureStaging(SimlodContext* ctx, uint64_t bytes) {
    bytes = (bytes + 255) & ~255ull;                         // every slot 256-byte aligned: full decode tiles take the TMA path
    if (ctx->staging && ctx->stagingSlotBytes >= bytes) return SIMLOD_OK;
    CU(D(cuStreamSynchronize)(ctx->streamCopy));
    CU(D(cuStreamSynchronize)(ctx->streamUpload));
    if (ctx->staging) { CU(D(cuMemFree)(ctx->staging)); ctx->staging = 0; }
    ctx->stagingSlots = (uint32_t)std::max<uint64_t>(2, std::min<uint64_t>(ctx->MAX_STAGING_SLOTS, (512ull << 20) / bytes));
    CU(D(cuMemAlloc)(&ctx->staging, (size_t)(bytes * ctx->stagingSlots)));
    ctx->stagingSlotBytes = bytes;
    ctx->stagingNext = 0;
    return SIMLOD_OK;
}

// Upload `count` LAS records and decode them into the next ring slot, then publish it. Host records are copied into the
// next staging slot on streamCopy (`copied`, if given, is recorded there once the host buffer has been read); the decode
// on streamUpload waits for that copy only, so copies of later batches do not queue behind a decode that waits for the
// SMs an update launch occupies.
static int uploadLasCommon(SimlodContext* ctx, const void* host, CUdeviceptr dev, uint32_t count, const SimlodLasLayout* layout,
                           CUevent copied = nullptr) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!layout) return fail(SIMLOD_ERR_INVALID, "null layout");
    uint32_t offsetRgb = 0;
    rc = lasRgbOffset(layout->format, layout->bytes_per_point, &offsetRgb); if (rc) return rc;
    uint32_t slot = 0;
    CUdeviceptr dst = 0;
    rc = claimSlot(ctx, count, &slot, &dst); if (rc) return rc;
    if (count) {
        CUdeviceptr records = dev;
        uint32_t s = 0;
        if (host) {
            rc = ensureStaging(ctx, SLOT_POINTS * layout->bytes_per_point); if (rc) return rc;
            s = ctx->stagingNext++ % ctx->stagingSlots;
            records = ctx->staging + (uint64_t)s * ctx->stagingSlotBytes;
            CU(D(cuStreamWaitEvent)(ctx->streamCopy, ctx->evStagingFree[s], 0));
            CU(D(cuMemcpyHtoDAsync)(records, host, (size_t)count * layout->bytes_per_point, ctx->streamCopy));
            if (copied) CU(D(cuEventRecord)(copied, ctx->streamCopy));
            CU(D(cuEventRecord)(ctx->evStaged[s], ctx->streamCopy));
            CU(D(cuStreamWaitEvent)(ctx->streamUpload, ctx->evStaged[s], 0));
        }
        uint64_t numPoints = count;
        uint32_t bpp = layout->bytes_per_point;
        double sx = layout->scale[0], sy = layout->scale[1], sz = layout->scale[2];
        double ox = layout->offset[0] + layout->translation[0], oy = layout->offset[1] + layout->translation[1], oz = layout->offset[2] + layout->translation[2];   // LasLoader.cpp:199-201
        unsigned blocks = (unsigned)std::min<uint64_t>((count + 255) / 256, (uint64_t)ctx->numSMs * 8);
        rc = launch(ctx, ctx->fn[K_LAS], blocks, 256, ctx->streamUpload, records, numPoints, bpp, offsetRgb, sx, sy, sz, ox, oy, oz, dst);
        if (rc) return rc;
        if (host) CU(D(cuEventRecord)(ctx->evStagingFree[s], ctx->streamUpload));
    } else if (copied) {
        CU(D(cuEventRecord)(copied, ctx->streamCopy));
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
    rc = launchConstruct(ctx, ctx->evStart, ctx->evEnd); if (rc) return rc;
    CU(D(cuEventSynchronize)(ctx->evEnd));
    if (kernel_ms) CU(D(cuEventElapsedTime)(kernel_ms, ctx->evStart, ctx->evEnd));
    rc = readStats(ctx); if (rc) return rc;
    return checkOverflow(ctx);
}

// How the batches of one insertion call become available to kernel_construct (insertBatches).
struct Feed {
    uint32_t gate = 20;        // launch once this many published batches await a launch; all of them once !more
    bool more = false;         // step can publish further batches before the device has consumed the published ones
    bool timed = true;         // *kernel_ms and *total_ms cover the launches from here on
    CUdeviceptr points = 0;    // kernel_construct's points argument (0: the ring)
    std::function<int(bool& progress)> step;   // copies and publishes what it can; sets progress if it did
};

// The main loop's streaming behaviour (main.cpp:1176-1180 + the uploader thread, :963-1063) without a frame in between:
// the feed publishes batches as far as the 50-slot ring allows and update launches go through the launch queue back to
// back (each consumes at most 20 batches or 10 ms, voxels.cu:22,883,940). A launch starts once the batches it is meant
// to consume are published, instead of snapshotting a half-filled ring.
static int insertBatches(SimlodContext* ctx, uint64_t numBatches, Feed& feed, float* kernel_ms, float* total_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    rc = readStats(ctx); if (rc) return rc;
    SimlodContext::LaunchQueue& q = ctx->queue;
    q.head = q.size = q.stalled = 0;
    const uint32_t target = ctx->uploaded + (uint32_t)numBatches;
    uint32_t covered = ctx->processed;                       // batches the enqueued launches are expected to have consumed
    bool timing = false;
    auto startTiming = [&]() -> int {
        timing = true;
        q.kernelMs = 0.0f;
        CU(D(cuEventRecord)(ctx->evTotalStart, ctx->streamMain));
        return SIMLOD_OK;
    };
    if (feed.timed) { rc = startTiming(); if (rc) return rc; }
    while (ctx->processed < target) {
        bool progress = false;
        rc = feed.step(progress); if (rc) return rc;
        if (feed.timed && !timing) { rc = startTiming(); if (rc) return rc; }
        if (q.size == 0) covered = std::min(covered, ctx->processed);   // a launch ran into its 10 ms budget: the rest is launched again
        while (q.size < q.DEPTH && ctx->uploaded > covered && (ctx->uploaded - covered >= feed.gate || !feed.more)) {
            const uint32_t take = std::min<uint32_t>(20u, ctx->uploaded - covered);
            rc = enqueueLaunch(ctx, covered + take, feed.points); if (rc) return rc;
            covered += take;
            progress = true;
        }
        while ((rc = retireLaunch(ctx, false)) == 1) progress = true;
        if (rc < 0) return rc;
        if (!progress) { rc = retireLaunch(ctx, true); if (rc < 0) return rc; }
    }
    while (q.size > 0) { rc = retireLaunch(ctx, true); if (rc < 0) return rc; }
    if (!timing) { rc = startTiming(); if (rc) return rc; }
    CU(D(cuEventRecord)(ctx->evTotalEnd, ctx->streamMain));
    CU(D(cuEventSynchronize)(ctx->evTotalEnd));
    if (kernel_ms) *kernel_ms = q.kernelMs;
    if (total_ms) CU(D(cuEventElapsedTime)(total_ms, ctx->evTotalStart, ctx->evTotalEnd));
    return SIMLOD_OK;
}

// Ring copy: the batches are copied into the ring as back-pressure allows. A host source arrives at PCIe speed, slower
// than the builder: it is published every 2 batches as it goes and launched from 2 batches on, so that insertion trails
// the upload closely. A device source arrives far faster than it is consumed: full 20-batch launches.
static int insertRing(SimlodContext* ctx, const SimlodPoint* host, CUdeviceptr dev, uint64_t count, float* kernel_ms, float* total_ms) {
    const uint64_t numBatches = (count + SLOT_POINTS - 1) / SLOT_POINTS;
    uint64_t next = 0;
    Feed feed;
    feed.gate = host ? 2u : 20u;
    feed.step = [&](bool& progress) -> int {
        for (; next < numBatches && ctx->uploaded - ctx->processed < RING_SLOTS; next++) {
            const uint64_t first = next * SLOT_POINTS;
            const uint32_t n = (uint32_t)std::min<uint64_t>(SLOT_POINTS, count - first);
            int rc = uploadCommon(ctx, host ? host + first : nullptr, host ? 0 : dev + first * sizeof(SimlodPoint), n, false);
            if (rc) return rc;
            progress = true;
            if (host && ctx->unpublished >= feed.gate) { rc = publishPending(ctx); if (rc) return rc; }
        }
        feed.more = next < numBatches;
        return publishPending(ctx);
    };
    return insertBatches(ctx, numBatches, feed, kernel_ms, total_ms);
}

int simlod_insert(SimlodContext* ctx, const SimlodPoint* host_points, uint64_t count, float* kernel_ms, float* total_ms) {
    if (!host_points && count) return fail(SIMLOD_ERR_INVALID, "null points");
    return insertRing(ctx, host_points, 0, count, kernel_ms, total_ms);
}

// A 16-byte aligned device-resident source is a zero-copy window: the point set already IS a sequence of 1 000 000-point
// batches in HBM, so copying it into the ring would only move 16 B/point a second time — and those device-to-device
// copies cannot run under the persistent cooperative kernel (measured: every launch waited 0.24 ms for the 20 copies
// behind it, tools/launch_gaps.py). kernel_construct addresses batch g as points + (g % 50) * 1 000 000
// (voxels.cu:886-889); within one window of 50 consecutive batches that is a linear map of g, so the launches of a window
// get a `points` argument that makes slot g % 50 land on batch g of the caller's buffer. The ring protocol is unchanged
// from the kernel's side (sizes and counter are published per window, the next window only after the device has
// consumed the current one); only the bytes do not move. An unaligned buffer goes through the ring: the kernel loads
// points 16 bytes at a time.
int simlod_insert_device(SimlodContext* ctx, uint64_t device_points, uint64_t count, float* kernel_ms, float* total_ms) {
    if (!device_points && count) return fail(SIMLOD_ERR_INVALID, "null points");
    if (!ctx) return fail(SIMLOD_ERR_INVALID, "null context");
    const CUdeviceptr dev = (CUdeviceptr)device_points;
    if ((dev & 15ull) != 0) return insertRing(ctx, nullptr, dev, count, kernel_ms, total_ms);
    const uint64_t numBatches = (count + SLOT_POINTS - 1) / SLOT_POINTS;
    const uint32_t g0 = ctx->uploaded;                      // global index of this call's first batch
    const uint32_t target = g0 + (uint32_t)numBatches;
    Feed feed;
    feed.timed = false;         // batches uploaded before the call sit in the real ring: they are consumed first, untimed
    feed.step = [&](bool& progress) -> int {
        if (ctx->queue.size > 0 || ctx->uploaded != ctx->processed || ctx->uploaded == target) return SIMLOD_OK;
        // the window is consumed: publish the next one (sizes + counter only)
        const uint32_t window = ctx->processed / (uint32_t)RING_SLOTS;
        const uint32_t windowEnd = std::min<uint32_t>(target, (window + 1u) * (uint32_t)RING_SLOTS);
        while (ctx->uploaded < windowEnd) {
            const uint64_t first = (uint64_t)(ctx->uploaded - g0) * SLOT_POINTS;
            ctx->hostSizes[ctx->uploaded % RING_SLOTS] = (uint32_t)std::min<uint64_t>(SLOT_POINTS, count - first);
            ctx->uploaded++;
            ctx->unpublished++;
        }
        // slot s of this window = batch window * 50 + s = the caller's batch (window * 50 + s - g0)
        feed.points = dev + (uint64_t)((int64_t)window * (int64_t)RING_SLOTS - (int64_t)g0) * (SLOT_POINTS * sizeof(SimlodPoint));
        feed.timed = true;
        progress = true;
        return publishPending(ctx);
    };
    return insertBatches(ctx, numBatches, feed, kernel_ms, total_ms);
}

// ---- streaming front end (SURVEY.md §8f-1, §8f-2) --------------------------------------------------------
}  // extern "C"

namespace {

constexpr uint64_t POOL_BYTES = 32ull * SLOT_POINTS * sizeof(SimlodPoint);    // 512 MB page-locked (the reference: 200 x 16 MB, main.cpp:35)
constexpr uint64_t MAX_POOL_SLOTS = 32;                                        // evPool[]
constexpr uint64_t PIECE_BYTES = 1ull << 20;                                   // loaders' unit of work: a multiple of 16

// One validated input of the streamer: where its records start, how many there are and how large, its box, and for LAS
// the decode layout (its translation is set once the union box is known). Owns its file descriptor.
struct StreamFile {
    std::string path;
    bool las = false;
    uint64_t dataOffset = 24, numPoints = 0;
    uint32_t bpp = sizeof(SimlodPoint);
    float min[3] = {}, max[3] = {};
    SimlodLasLayout layout{};
    int fd = -1;
    bool direct = false;           // fd was opened with O_DIRECT
};
struct StreamFiles {
    std::vector<StreamFile> v;
    ~StreamFiles() { for (StreamFile& f : v) if (f.fd >= 0) close(f.fd); }
};
// batch k of a streamed list: `count` records of file `file` from its record `first` on (main.cpp:711-720, 737-745)
struct StreamBatch { uint32_t file; uint64_t first; uint32_t count; };

uint64_t fileSizeOf(const char* path) {
    struct stat st;
    return stat(path, &st) == 0 ? (uint64_t)st.st_size : 0;
}

bool iEndsWith(const std::string& s, const char* suffix) {         // iEndsWith of the reference's unsuck.hpp
    const size_t n = strlen(suffix);
    if (s.size() < n) return false;
    for (size_t i = 0; i < n; i++) if (tolower((unsigned char)s[s.size() - n + i]) != tolower((unsigned char)suffix[i])) return false;
    return true;
}

int readLasHeader(const char* path, SimlodLasHeader* h) {          // loadHeader, LasLoader.h:21-55
    FILE* f = fopen(path, "rb");
    if (!f) return fail(SIMLOD_ERR_INVALID, "cannot open %s", path);
    unsigned char b[375] = {0};
    const size_t got = fread(b, 1, sizeof(b), f);
    fclose(f);
    if (got < 4 || memcmp(b, "LASF", 4) != 0) return fail(SIMLOD_ERR_INVALID, "%s is not a LAS file (no LASF signature)", path);
    if (got < 227) return fail(SIMLOD_ERR_INVALID, "%s is shorter than a LAS header (%zu bytes)", path, got);
    auto u16 = [&](int o) { uint16_t v; memcpy(&v, b + o, 2); return (uint32_t)v; };
    auto u32 = [&](int o) { uint32_t v; memcpy(&v, b + o, 4); return v; };
    auto f64 = [&](int o) { double v; memcpy(&v, b + o, 8); return v; };
    memset(h, 0, sizeof(*h));
    h->version_major = b[24];
    h->version_minor = b[25];
    h->header_size = u16(94);
    h->offset_to_point_data = u32(96);
    h->format = b[104];
    h->bytes_per_point = u16(105);
    if (h->version_major == 1 && h->version_minor <= 3) {
        h->num_points = u32(107);
    } else {
        if (got < 255) return fail(SIMLOD_ERR_INVALID, "%s is shorter than a LAS %u.%u header (%zu bytes)", path, h->version_major, h->version_minor, got);
        memcpy(&h->num_points, b + 247, 8);
    }
    for (int i = 0; i < 3; i++) {
        h->scale[i] = f64(131 + 8 * i);
        h->offset[i] = f64(155 + 8 * i);
        h->min[i] = f64(187 + 16 * i);
        h->max[i] = f64(179 + 16 * i);
    }
    return SIMLOD_OK;
}

int probeSimlod(const char* path, StreamFile* out) {
    FILE* f = fopen(path, "rb");
    if (!f) return fail(SIMLOD_ERR_INVALID, "cannot open %s", path);
    float hdr[6];
    const size_t got = fread(hdr, 1, sizeof(hdr), f);
    fclose(f);
    const uint64_t size = fileSizeOf(path);
    if (got != sizeof(hdr) || size < 24) return fail(SIMLOD_ERR_INVALID, "%s is not a .simlod file (shorter than its 24-byte header)", path);
    out->path = path;
    out->numPoints = (size - 24) / 16;                             // main.cpp:738
    for (int i = 0; i < 3; i++) { out->min[i] = hdr[i]; out->max[i] = hdr[3 + i]; }
    return SIMLOD_OK;
}

int probeLas(const char* path, StreamFile* out) {
    SimlodLasHeader h;
    int rc = readLasHeader(path, &h); if (rc) return rc;
    uint32_t offsetRgb = 0;
    rc = lasRgbOffset(h.format, h.bytes_per_point, &offsetRgb, path); if (rc) return rc;
    const uint64_t size = fileSizeOf(path);
    if (h.offset_to_point_data > size || h.num_points > (size - h.offset_to_point_data) / h.bytes_per_point)
        return fail(SIMLOD_ERR_INVALID, "%s: %llu records of %u bytes from byte %u run past the end of the %llu-byte file", path,
                    (unsigned long long)h.num_points, h.bytes_per_point, h.offset_to_point_data, (unsigned long long)size);
    out->path = path;
    out->las = true;
    out->dataOffset = h.offset_to_point_data;
    out->numPoints = h.num_points;
    out->bpp = h.bytes_per_point;
    for (int i = 0; i < 3; i++) {
        out->min[i] = (float)h.min[i];                             // main.cpp:700-709
        out->max[i] = (float)h.max[i];
        out->layout.scale[i] = h.scale[i];
        out->layout.offset[i] = h.offset[i];
    }
    out->layout.bytes_per_point = h.bytes_per_point;
    out->layout.format = h.format;
    return SIMLOD_OK;
}

// the streamer's page-locked pool (POOL_BYTES) and its slot events, allocated on first use
int ensurePinnedPool(SimlodContext* ctx) {
    if (ctx->pinnedPool) return SIMLOD_OK;
    NumaLocal onGpuNode(ctx);
    CU(D(cuMemHostAlloc)(&ctx->pinnedPool, (size_t)POOL_BYTES, CU_MEMHOSTALLOC_PORTABLE));
    for (uint64_t i = 0; i < MAX_POOL_SLOTS; i++) CU(D(cuEventCreate)(&ctx->evPool[i], CU_EVENT_DISABLE_TIMING));
    return SIMLOD_OK;
}

int openForStream(StreamFile* f, bool direct) {
    // SIMLOD_STREAM_DIRECT: unbuffered reads, as the reference's Windows loader does (SimlodLoader.cpp:59-141, FILE_FLAG_NO_BUFFERING):
    // whole 4 KB blocks straight from the device into a per-thread block buffer — no page-cache copy, no cache pollution —
    // for files that are not resident in the page cache (a cold 5.6 GB scan gains nothing from being cached on the way)
    f->fd = open(f->path.c_str(), direct ? (O_RDONLY | O_DIRECT) : O_RDONLY);
    if (f->fd < 0) return fail(SIMLOD_ERR_INVALID, direct ? "cannot open %s with O_DIRECT (tmpfs and some overlay file systems do not support it)" : "cannot open %s", f->path.c_str());
    f->direct = direct;
    return SIMLOD_OK;
}

// One entry of a file list: the path must exist and name a .las or .simlod file, whose header is read and checked
int probeListedFile(const char* p, uint32_t i, StreamFile* f) {
    if (!p) return fail(SIMLOD_ERR_INVALID, "null path at list position %u", i);
    struct stat st;
    if (stat(p, &st) != 0) return fail(SIMLOD_ERR_INVALID, "%s does not exist", p);
    const std::string s(p);
    if (iEndsWith(s, ".laz")) return fail(SIMLOD_ERR_INVALID, "%s: LAZ is not supported", p);
    if (iEndsWith(s, ".las")) return probeLas(p, f);
    if (iEndsWith(s, ".simlod")) return probeSimlod(p, f);
    return fail(SIMLOD_ERR_INVALID, "%s: unsupported file type (expected .las or .simlod)", p);
}

// the union of the files' boxes (main.cpp:700-709, 724-733, 763-765)
void unionBox(const StreamFiles& files, float bmin[3], float bmax[3]) {
    for (int i = 0; i < 3; i++) { bmin[i] = std::numeric_limits<float>::infinity(); bmax[i] = -bmin[i]; }
    for (const StreamFile& f : files.v)
        for (int a = 0; a < 3; a++) { bmin[a] = std::min(bmin[a], f.min[a]); bmax[a] = std::max(bmax[a], f.max[a]); }
}

}  // namespace

extern "C" {

// reload() + spawnLoader + spawnUploader (main.cpp:644-773, 811-958, 963-1063) over validated files: the union box sets the
// uniforms, the octree is reset, and the files' batches stream through the pinned pool in list order.
static int streamFiles(SimlodContext* ctx, StreamFiles& files, int loader_threads, uint64_t* num_points, float* kernel_ms, float* total_ms) {
    // the box (main.cpp:700-709, 724-733, 763-765) and the batch list (main.cpp:711-720, 737-745)
    float bmin[3], bmax[3];
    unionBox(files, bmin, bmax);
    std::vector<StreamBatch> batches;
    uint64_t numPoints = 0;
    uint32_t maxBpp = 0, maxLasBpp = 0;
    for (uint32_t i = 0; i < (uint32_t)files.v.size(); i++) {
        const StreamFile& f = files.v[i];
        for (uint64_t first = 0; first < f.numPoints; first += SLOT_POINTS)
            batches.push_back({i, first, (uint32_t)std::min<uint64_t>(SLOT_POINTS, f.numPoints - first)});
        numPoints += f.numPoints;
        if (f.numPoints) maxBpp = std::max(maxBpp, f.bpp);
        if (f.numPoints && f.las) maxLasBpp = std::max(maxLasBpp, f.bpp);
    }
    for (StreamFile& f : files.v)
        for (int a = 0; a < 3; a++) f.layout.translation[a] = (double)(-bmin[a]);          // main.cpp:868
    const uint64_t numBatches = batches.size();
    if (num_points) *num_points = numPoints;
    for (int i = 0; i < 3; i++) { ctx->uniforms.boxMin[i] = 0.0f; ctx->uniforms.boxMax[i] = bmax[i] - bmin[i]; }   // main.cpp:312-313
    int rc = simlod_reset(ctx); if (rc) return rc;                        // reload() -> reset
    rc = ensurePinnedPool(ctx); if (rc) return rc;
    if (maxLasBpp) { rc = ensureStaging(ctx, SLOT_POINTS * maxLasBpp); if (rc) return rc; }
    // a pool slot holds one batch of the largest records in the list: 32 slots of 16 MB for .simlod points, 5 of 96 MB
    // for the largest LAS records. SLOT_POINTS * bpp is a multiple of 16, so every slot and piece starts 16-byte aligned.
    const uint64_t slotBytes = SLOT_POINTS * std::max<uint32_t>(maxBpp, 16);
    const uint64_t poolSlots = std::min<uint64_t>(MAX_POOL_SLOTS, POOL_BYTES / slotBytes);
    // loaders: batch k goes to pool slot k % poolSlots once the copy of batch k - poolSlots has left it. The unit of work
    // is a 1 MB piece of a batch's file bytes, handed out in list order, so that all threads read the batch the uploader
    // needs next (the reference reads one whole batch per thread, main.cpp:811-958: every batch then arrives late).
    const uint64_t PIECES = (slotBytes + PIECE_BYTES - 1) / PIECE_BYTES;
    const bool trace = getenv("SIMLOD_STREAM_TRACE") != nullptr;          // developer aid: host timeline to stderr
    const auto tBegin = std::chrono::steady_clock::now();
    auto since = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tBegin).count(); };
    double tSpawned = 0, tFirst = 0, tAllLoaded = 0, tLastUpload = 0, tJoined = 0;
    std::vector<std::atomic<int>> loaded(numBatches);          // pieces of batch k that have arrived
    for (auto& l : loaded) l.store(0);
    std::atomic<int64_t> copiesDone{0};           // batches whose host->device copy has completed
    std::atomic<uint64_t> nextPiece{0};
    std::atomic<bool> abort{false};
    std::atomic<int> badFile{-1};                 // the file a read failed in
    const int nThreads = std::max(1, std::min(loader_threads, 64));
    if (!ctx->loaderPool) ctx->loaderPool = new LoaderPool();
    LoaderPool* pool = ctx->loaderPool;
    pool->run(nThreads, [&, pool](int worker) {
        for (;;) {
            const uint64_t item = nextPiece.fetch_add(1);
            const uint64_t k = item / PIECES, piece = item % PIECES;
            if (k >= numBatches || abort.load()) break;
            while (copiesDone.load() + (int64_t)poolSlots <= (int64_t)k && !abort.load()) std::this_thread::yield();
            const StreamBatch& b = batches[k];
            const StreamFile& f = files.v[b.file];
            const uint64_t inBatch = (uint64_t)b.count * f.bpp, p0 = piece * PIECE_BYTES;
            if (p0 < inBatch) {
                uint64_t bytes = std::min<uint64_t>(PIECE_BYTES, inBatch - p0);
                char* dst = (char*)ctx->pinnedPool + (k % poolSlots) * slotBytes + p0;
                off_t at = (off_t)(f.dataOffset + b.first * f.bpp + p0);
                // only the last piece of a batch can end off a 16-byte boundary: its streaming copy rounds up, into the
                // slot's own bytes (round16(count * bpp) <= SLOT_POINTS * bpp <= slotBytes), and those bytes are not uploaded
                bool ok = true;
                if (f.direct) {
                    // the piece is <= 1 MB at any file offset: read the 4 KB blocks that cover it
                    char* blockBuf = pool->directBuffer(worker);
                    const off_t a0 = at & ~(off_t)4095;
                    const size_t want = (size_t)((((uint64_t)at + bytes + 4095ull) & ~4095ull) - (uint64_t)a0);
                    size_t have = 0;
                    while (have < want) {
                        ssize_t r = pread(f.fd, blockBuf + have, want - have, a0 + (off_t)have);
                        if (r < 0) { ok = false; break; }
                        if (r == 0) break;                                        // end of file inside the last block
                        have += (size_t)r;
                        if (r % 4096) break;                                      // short read at the end of the file
                    }
                    if (have < (size_t)(at - a0) + bytes) ok = false;
                    else copyStreamingU(dst, blockBuf + (at - a0), (bytes + 15) & ~15ull);
                    bytes = 0;
                }
                char* stage = pool->bounce[worker];
                while (ok && bytes) {
                    uint64_t want = std::min<uint64_t>(bytes, LoaderPool::BOUNCE_BYTES), have = 0;
                    while (have < want) {
                        ssize_t r = pread(f.fd, stage + have, want - have, at + (off_t)have);
                        if (r <= 0) { ok = false; break; }
                        have += (uint64_t)r;
                    }
                    if (!ok) break;
                    copyStreaming(dst, stage, (want + 15) & ~15ull);
                    dst += want; at += (off_t)want; bytes -= want;
                }
                if (!ok) { int none = -1; badFile.compare_exchange_strong(none, (int)b.file); abort.store(true); }
            }
            loaded[k].fetch_add(1);
        }
    });
    const int allPieces = (int)PIECES;
    tSpawned = since();
    // stops and joins the loader threads on every exit; joined early once the last batch is uploaded (the files are
    // closed by StreamFiles, after this)
    struct Loaders {
        LoaderPool* pool; std::atomic<bool>& abort; bool joined = false;
        void join() { if (joined) return; abort.store(true); pool->wait(); joined = true; }
        ~Loaders() { join(); }
    } loaders{pool, abort};

    // uploader: a batch goes to the ring once all its pieces have loaded, one batch per step, and a launch follows every
    // 2 batches; its pool slot goes back to the loaders when the copy out of it has completed (evPool, in order).
    // .simlod points are copied into their ring slot; LAS records into a device staging slot on the copy stream and
    // decoded into the ring slot (uploadLasCommon).
    uint64_t next = 0;
    int64_t copiesEnqueued = 0;
    auto recycle = [&]() {
        while (copiesDone.load() < copiesEnqueued && D(cuEventQuery)(ctx->evPool[copiesDone.load() % poolSlots]) == CUDA_SUCCESS) copiesDone.fetch_add(1);
    };
    Feed feed;
    feed.gate = 2;
    feed.more = numBatches > 0;
    feed.step = [&](bool& progress) -> int {
        if (next == numBatches || ctx->uploaded - ctx->processed >= RING_SLOTS) return SIMLOD_OK;
        while (loaded[next].load() < allPieces && !abort.load()) std::this_thread::yield();
        if (abort.load()) {
            const int bad = badFile.load();
            return fail(SIMLOD_ERR_INVALID, "read error in %s", files.v[bad >= 0 ? bad : batches[next].file].path.c_str());
        }
        if (next == 0) tFirst = since();
        if (next + 1 == numBatches) tAllLoaded = since();
        const StreamBatch& b = batches[next];
        const StreamFile& f = files.v[b.file];
        char* src = (char*)ctx->pinnedPool + (next % poolSlots) * slotBytes;
        CUevent copied = ctx->evPool[next % poolSlots];
        if (f.las) {
            int urc = uploadLasCommon(ctx, src, 0, b.count, &f.layout, copied); if (urc) return urc;
        } else {
            int urc = uploadCommon(ctx, src, 0, b.count); if (urc) return urc;
            CU(D(cuEventRecord)(copied, ctx->streamUpload));
        }
        copiesEnqueued++;
        recycle();
        // when all pool slots are in flight, wait for the oldest copy instead of spinning on the loaders
        if (copiesEnqueued - copiesDone.load() >= (int64_t)poolSlots) { CU(D(cuEventSynchronize)(ctx->evPool[copiesDone.load() % poolSlots])); recycle(); }
        progress = true;
        feed.more = ++next < numBatches;
        if (!feed.more) { tLastUpload = since(); loaders.join(); tJoined = since(); }
        return SIMLOD_OK;
    };
    rc = insertBatches(ctx, numBatches, feed, kernel_ms, total_ms); if (rc) return rc;
    if (trace) fprintf(stderr, "[simlod stream] %zu files, %llu batches, %d threads: started %.2f ms, first batch %.2f, all loaded %.2f, last upload enqueued %.2f, loaders idle %.2f, done %.2f\n",
                       files.v.size(), (unsigned long long)numBatches, nThreads, tSpawned, tFirst, tAllLoaded, tLastUpload, tJoined, since());
    return SIMLOD_OK;
}

int simlod_insert_simlod_file(SimlodContext* ctx, const char* path, int loader_threads, uint64_t* num_points,
                              float* kernel_ms, float* total_ms) {
    return simlod_insert_simlod_file_ex(ctx, path, loader_threads, 0, num_points, kernel_ms, total_ms);
}

int simlod_insert_simlod_file_ex(SimlodContext* ctx, const char* path, int loader_threads, uint32_t flags, uint64_t* num_points,
                                 float* kernel_ms, float* total_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!path) return fail(SIMLOD_ERR_INVALID, "null path");
    StreamFiles files;
    files.v.emplace_back();
    rc = probeSimlod(path, &files.v[0]); if (rc) return rc;
    rc = openForStream(&files.v[0], (flags & SIMLOD_STREAM_DIRECT) != 0); if (rc) return rc;
    return streamFiles(ctx, files, loader_threads, num_points, kernel_ms, total_ms);
}

int simlod_read_las_header(const char* path, SimlodLasHeader* out) {
    if (!path || !out) return fail(SIMLOD_ERR_INVALID, "null argument");
    return readLasHeader(path, out);
}

int simlod_insert_files(SimlodContext* ctx, const char* const* paths, uint32_t num_paths, int loader_threads,
                        uint32_t flags, uint64_t* num_points, float* kernel_ms, float* total_ms) {
    if (!paths || num_paths == 0) return fail(SIMLOD_ERR_INVALID, "empty file list");
    // every path, header and size is checked, and every file opened, before the context is touched
    int rc = SIMLOD_OK;
    StreamFiles files;
    files.v.resize(num_paths);
    for (uint32_t i = 0; i < num_paths; i++) {
        rc = probeListedFile(paths[i], i, &files.v[i]); if (rc) return rc;
        rc = openForStream(&files.v[i], (flags & SIMLOD_STREAM_DIRECT) != 0); if (rc) return rc;
    }
    rc = setCurrent(ctx); if (rc) return rc;
    return streamFiles(ctx, files, loader_threads, num_points, kernel_ms, total_ms);
}

int simlod_files_box(const char* const* paths, uint32_t num_paths, float box_min[3], float box_max[3]) {
    if (!paths || num_paths == 0) return fail(SIMLOD_ERR_INVALID, "empty file list");
    if (!box_min || !box_max) return fail(SIMLOD_ERR_INVALID, "null argument");
    StreamFiles files;
    files.v.resize(num_paths);
    for (uint32_t i = 0; i < num_paths; i++) { int rc = probeListedFile(paths[i], i, &files.v[i]); if (rc) return rc; }
    unionBox(files, box_min, box_max);
    return SIMLOD_OK;
}

int simlod_render(SimlodContext* ctx, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    SimlodUniforms u = ctx->uniforms;
    u.frameCounter = ctx->frameCounter++;
    CUdeviceptr rb = ctx->buf.renderbuffer, nodes = ctx->buf.nodes, stats = ctx->buf.stats, frameStart = ctx->frameStart, cudaprint = ctx->cudaprint;
    CUsurfObject surf = ctx->surface;
    const Program& program = ctx->programs[SIMLOD_PROGRAM_RENDER];
    const bool clipped = ctx->clip.mode != SIMLOD_CLIP_NONE;
    if (clipped && !program.fnClip) return fail(SIMLOD_ERR_MODULE, "a clip is set and the render module does not export simlod_render_clip");
    SimlodClip clip = ctx->clip;
    CU(D(cuEventRecord)(ctx->evStart, ctx->streamMain));
    if (clipped) rc = launchCooperative(ctx, program.fnClip, ctx->renderBlocks, 256, ctx->streamMain, rb, u, nodes, surf, stats, frameStart, cudaprint, clip);
    else rc = launchCooperative(ctx, program.fn, ctx->renderBlocks, 256, ctx->streamMain,
                                rb, u, nodes, surf, stats, frameStart, cudaprint);     // main.cpp:499-507
    if (rc) return rc;
    CU(D(cuEventRecord)(ctx->evEnd, ctx->streamMain));
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
    CU(D(cuMemcpyDtoH)(out, ctx->buf.renderbuffer + rbuf::OFF_FB, (size_t)ctx->cfg.width * ctx->cfg.height * 8));
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
    rc = launch(ctx, ctx->fn[K_RCP], 1, 1, ctx->streamMain, x, dst); if (rc) return rc;
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
    if (kind == SIMLOD_GEN_UNIFORM)
        rc = launch(ctx, ctx->fn[K_GEN_UNIFORM], blocks, 256, ctx->streamMain, dst, first, count, seed, size);
    else if (kind == SIMLOD_GEN_TERRAIN || kind == SIMLOD_GEN_SHELL)
        rc = launch(ctx, ctx->fn[kind == SIMLOD_GEN_TERRAIN ? K_GEN_TERRAIN : K_GEN_SHELL], blocks, 256, ctx->streamMain, dst, n_total, first, count, seed);
    else
        return fail(SIMLOD_ERR_INVALID, "unknown generator %d", kind);
    if (rc) return rc;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    return SIMLOD_OK;
}

int simlod_synchronize(SimlodContext* ctx) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CU(D(cuStreamSynchronize)(ctx->streamCopy));
    CU(D(cuStreamSynchronize)(ctx->streamUpload));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    return SIMLOD_OK;
}

int simlod_flush_l2(SimlodContext* ctx) {
    int rc = setCurrent(ctx); if (rc) return rc;
    CUdeviceptr dst = ctx->flushBuf;
    uint64_t count = L2_FLUSH_BYTES / 16;
    uint32_t value = 0;
    rc = launch(ctx, ctx->fn[K_FILL], (unsigned)(ctx->numSMs * 8), 256, ctx->streamMain, dst, count, value); if (rc) return rc;
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    return SIMLOD_OK;
}

// ---- octree export (DESIGN.md §9.4, §9.5); kernels in export.cu --------------------------------------------
namespace {
constexpr uint64_t align16(uint64_t v) { return (v + 15) & ~15ull; }
constexpr size_t CTL_HOST_BYTES = 128;      // the pinned copy of the control word
static_assert(sizeof(ExportCtl) <= CTL_HOST_BYTES && sizeof(QueryCtl) <= CTL_HOST_BYTES && sizeof(NearestCtl) <= CTL_HOST_BYTES &&
              sizeof(RayCtl) <= CTL_HOST_BYTES && sizeof(NearestCtl) + sizeof(RadiusCtl) <= CTL_HOST_BYTES &&
              sizeof(HeightmapCtl) <= CTL_HOST_BYTES, "pinned control word");

// Consecutive 16-byte aligned regions of one allocation: take() returns the offset of the next one
struct Layout { uint64_t bytes = 0; uint64_t take(uint64_t n) { const uint64_t off = bytes; bytes += align16(n); return off; } };

// A control struct on the device and the host copy it is read into
struct CtlRead { CUdeviceptr src; void* dst; size_t bytes; };

// Up to four ordered marks on streamMain, on the context's four events; stage i is the time from mark i to mark i + 1.
// finish() makes the last mark, waits for it and reads the stages into ms[]. Control structs to read back are copied one
// after the other into the pinned control word behind the mark, and the wait is the one synchronisation of streamMain
// that brings them to their host copies; without them it waits on the mark's event.
struct StageClock {
    SimlodContext* ctx; CUevent ev[4]; int marks = 0;
    explicit StageClock(SimlodContext* c) : ctx(c), ev{c->evStart, c->evEnd, c->evTotalStart, c->evTotalEnd} {}
    int mark() {                            // the pinned control word is allocated before any stage is timed
        if (marks == 4) return fail(SIMLOD_ERR_INVALID, "internal: a stage clock has four marks");
        if (!ctx->hExportCtl) CU(D(cuMemHostAlloc)(&ctx->hExportCtl, CTL_HOST_BYTES, 0));
        CU(D(cuEventRecord)(ev[marks++], ctx->streamMain)); return SIMLOD_OK;
    }
    int finish(float* ms, std::initializer_list<CtlRead> reads = {}) {
        int rc = mark(); if (rc) return rc;
        uint8_t* const h = (uint8_t*)ctx->hExportCtl;
        size_t at = 0;
        for (const CtlRead& r : reads) { CU(D(cuMemcpyDtoHAsync)(h + at, r.src, r.bytes, ctx->streamMain)); at += r.bytes; }
        if (reads.size()) CU(D(cuStreamSynchronize)(ctx->streamMain)); else CU(D(cuEventSynchronize)(ev[marks - 1]));
        at = 0;
        for (const CtlRead& r : reads) { memcpy(r.dst, h + at, r.bytes); at += r.bytes; }
        for (int i = 0; i + 1 < marks; i++) CU(D(cuEventElapsedTime)(&ms[i], ev[i], ev[i + 1]));
        return SIMLOD_OK;
    }
};

// the refusal of a depth deeper than the octree's deepest level, for the entry point `what`
int checkDepth(const char* what, int32_t depth) {
    return depth > SIMLOD_MAX_DEPTH ? fail(SIMLOD_ERR_INVALID, "%s depth %d exceeds the octree's maximum depth %d", what, depth, (int)SIMLOD_MAX_DEPTH) : SIMLOD_OK;
}

// the refusal of the first address that is not a multiple of its alignment (or null, where one is required), for the
// entry point `what`
struct Aligned { const char* name; uint64_t addr; uint64_t align; bool required = false; };
int checkAligned(const char* what, std::initializer_list<Aligned> addrs) {
    for (const Aligned& a : addrs)
        if (a.addr % a.align || (a.required && !a.addr))
            return fail(SIMLOD_ERR_INVALID, "%s: %s must be %s%llu-byte aligned", what, a.name, a.required ? "a device address, " : "", (unsigned long long)a.align);
    return SIMLOD_OK;
}

// The context's export / query scratch, sized by its buffers: one record, node index and first item per node of nodes[],
// and one chunk item per chunk the heap can hold. The view adds per node a drawn byte, and per record a mark byte, an
// index and a second record and node index; the query adds one word per item. The control word comes last.
enum class ScratchUse { EXPORT, VIEW, QUERY };
struct Scratch {
    uint32_t maxRecords = 0;
    uint64_t itemsCap = 0;
    CUdeviceptr rec = 0, recNode = 0, recItem = 0, items = 0, words = 0, ctl = 0;
    ViewScratch view{};                     // all null unless VIEW
};
int scratchFor(SimlodContext* ctx, ScratchUse use, Scratch* s) {
    const uint64_t n = (uint64_t)(uint32_t)(ctx->buf.nodes_bytes / sizeof(SimlodNode));
    s->maxRecords = (uint32_t)n;
    s->itemsCap = ctx->buf.persistent_bytes / SIMLOD_CHUNK_STRIDE + 1;
    Layout l;
    const uint64_t rec = l.take(n * sizeof(SimlodExportNode)), recNode = l.take(n * 4), recItem = l.take(n * 8), items = l.take(s->itemsCap * 16);
    uint64_t drawn = 0, viewRec = 0, viewNode = 0, mark = 0, index = 0, words = 0;
    if (use == ScratchUse::VIEW) {
        drawn = l.take(n); mark = l.take(n); index = l.take(n * 4);
        viewRec = l.take(n * sizeof(SimlodExportNode)); viewNode = l.take(n * 4);
    }
    if (use == ScratchUse::QUERY) words = l.take(s->itemsCap * 8);
    const uint64_t ctl = l.take(use == ScratchUse::QUERY ? sizeof(QueryCtl) : sizeof(ExportCtl));
    int rc = growDevice(&ctx->exportScratch, &ctx->exportScratchBytes, l.bytes); if (rc) return rc;
    const CUdeviceptr base = ctx->exportScratch;
    s->rec = base + rec; s->recNode = base + recNode; s->recItem = base + recItem; s->items = base + items; s->ctl = base + ctl;
    s->words = use == ScratchUse::QUERY ? base + words : 0;
    if (use == ScratchUse::VIEW)
        s->view = ViewScratch{devPtr(base + drawn), devPtr(base + viewRec), devPtr(base + viewNode), devPtr(base + mark), devPtr(base + index)};
    return SIMLOD_OK;
}

// the message of ExportCtl::error, for the export and the query
int failInconsistent(uint32_t error) {
    return fail(SIMLOD_ERR_INVALID, "octree image is inconsistent (error %u: %u child pointer outside nodes[], %u chunk pointer outside the used heap, %u list shorter than its count, %u inner node without 8 children)",
                error, (uint32_t)EXPORT_ERR_CHILD, (uint32_t)EXPORT_ERR_CHUNK, (uint32_t)EXPORT_ERR_SHORT, (uint32_t)EXPORT_ERR_PARTIAL);
}

// the chunk-list walk of the export and the query, into scratch: one item per chunk of the planned records' lists
int launchCollect(SimlodContext* ctx, Scratch& s) {
    CUdeviceptr nodes = ctx->buf.nodes, heap = ctx->buf.persistent;
    uint64_t heapBytes = ctx->buf.persistent_bytes;
    return launch(ctx, ctx->fn[K_EXPORT_COLLECT], (unsigned)ctx->numSMs * 2, 256, ctx->streamMain,
                  nodes, heap, heapBytes, s.rec, s.recNode, s.recItem, s.items, s.itemsCap, s.ctl);
}

// Stage 1 of an export, into scratch only: the view's drawn flags, the plan and the chunk-list walk. On success p holds
// the checked ExportCtl and the scratch it describes.
struct ExportPlanned {
    Scratch s;
    ExportCtl c{};
    float ms = 0.0f;
};
int exportPlan(SimlodContext* ctx, int32_t depth, const SimlodUniforms* view, ExportPlanned* p, float* kernel_ms = nullptr) {
    struct Report { float* dst; const float& ms; ~Report() { if (dst) *dst = ms; } } report{kernel_ms, p->ms};   // on every return
    Scratch& s = p->s;
    int rc = scratchFor(ctx, view ? ScratchUse::VIEW : ScratchUse::EXPORT, &s); if (rc) return rc;
    CUdeviceptr nodes = ctx->buf.nodes, stats = ctx->buf.stats;
    // stage 1: the view's drawn flags (one thread per node), plan (one block) and the chunk-list walk, all into scratch only
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    if (view) {
        SimlodUniforms u = *view;
        rc = launch(ctx, ctx->fn[K_EXPORT_VIEW_FLAGS], (unsigned)ctx->numSMs * 4, 256, ctx->streamMain, nodes, stats, u, s.maxRecords, s.view.drawn);
        if (rc) return rc;
        rc = launch(ctx, ctx->fn[K_EXPORT_PLAN_VIEW], 1, 1024, ctx->streamMain, nodes, stats, s.maxRecords, s.rec, s.recNode, s.recItem, s.ctl, s.view);
    } else {
        rc = launch(ctx, ctx->fn[K_EXPORT_PLAN], 1, 1024, ctx->streamMain, nodes, stats, depth, s.maxRecords, s.rec, s.recNode, s.recItem, s.ctl);
    }
    if (rc) return rc;
    rc = launchCollect(ctx, s); if (rc) return rc;
    rc = clock.finish(&p->ms, {{s.ctl, &p->c, sizeof p->c}}); if (rc) return rc;
    if (p->c.error) return failInconsistent(p->c.error);
    return SIMLOD_OK;
}

// The fields NearestArgs, RadiusArgs, RayArgs and HeightmapArgs share: the plan's records and chunk items, the cut and the octree cube
extern "C++" template <class Args> Args planArgs(const ExportPlanned& p, const SimlodUniforms& u, int32_t depth) {
    Args a{};
    a.rec = devPtr(p.s.rec); a.recItem = devPtr(p.s.recItem); a.items = devPtr(p.s.items);
    a.numRecords = p.c.numNodes; a.depth = depth < 0 ? -1 : depth;
    std::copy_n(u.boxMin, 3, a.boxMin); std::copy_n(u.boxMax, 3, a.boxMax);
    return a;
}

// The export of simlod_export_octree (view == nullptr) and simlod_export_view (the LOD cut for *view).
int exportOctree(SimlodContext* ctx, int32_t depth, const SimlodUniforms* view, uint64_t dst_nodes, uint64_t node_capacity,
                 uint64_t dst_samples, uint64_t sample_capacity, SimlodExportInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!info) return fail(SIMLOD_ERR_INVALID, "null info");
    rc = checkDepth("export", depth); if (rc) return rc;
    rc = checkAligned("export", {{"dst_nodes", dst_nodes, 16}, {"dst_samples", dst_samples, 16}}); if (rc) return rc;
    ExportPlanned p;
    rc = exportPlan(ctx, depth, view, &p, kernel_ms); if (rc) return rc;
    const ExportCtl c = p.c;
    info->num_nodes = c.numNodes; info->max_level = c.maxLevel;
    info->num_samples = c.numSamples; info->num_points = c.numPoints; info->num_voxels = c.numVoxels;
    if (!dst_nodes && !dst_samples) return SIMLOD_OK;          // size query
    if (!dst_nodes || node_capacity < c.numNodes)
        return fail(SIMLOD_ERR_INVALID, "node destination holds %llu records, the export has %u", (unsigned long long)(dst_nodes ? node_capacity : 0), c.numNodes);
    if (c.numSamples && (!dst_samples || sample_capacity < c.numSamples))
        return fail(SIMLOD_ERR_INVALID, "sample destination holds %llu samples, the export has %llu", (unsigned long long)(dst_samples ? sample_capacity : 0), (unsigned long long)c.numSamples);
    // stage 2: gather into the destination
    CUdeviceptr dn = (CUdeviceptr)dst_nodes, ds = (CUdeviceptr)dst_samples;
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_EXPORT_GATHER], (unsigned)ctx->numSMs * 4, 256, ctx->streamMain, p.s.rec, dn, p.s.items, ds, p.s.ctl);
    if (rc) return rc;
    float gatherMs = 0.0f;
    rc = clock.finish(&gatherMs); if (rc) return rc;
    if (kernel_ms) *kernel_ms = p.ms + gatherMs;
    return SIMLOD_OK;
}
}  // namespace

int simlod_export_octree(SimlodContext* ctx, int32_t depth, uint64_t dst_nodes, uint64_t node_capacity,
                         uint64_t dst_samples, uint64_t sample_capacity, SimlodExportInfo* info, float* kernel_ms) {
    return exportOctree(ctx, depth, nullptr, dst_nodes, node_capacity, dst_samples, sample_capacity, info, kernel_ms);
}

int simlod_export_view(SimlodContext* ctx, uint64_t dst_nodes, uint64_t node_capacity, uint64_t dst_samples,
                       uint64_t sample_capacity, SimlodExportInfo* info, float* kernel_ms) {
    if (!ctx) return fail(SIMLOD_ERR_INVALID, "null context");
    return exportOctree(ctx, -1, &ctx->uniforms, dst_nodes, node_capacity, dst_samples, sample_capacity, info, kernel_ms);
}

// ---- region query (DESIGN.md §9.8); kernels in query.cu, the chunk-list walk is export.cu's ----------------------------
namespace {
int checkRegion(const SimlodRegion* r) {
    if (!r) return fail(SIMLOD_ERR_INVALID, "null region");
    auto finite = [](const float* v, int n) { for (int i = 0; i < n; i++) if (!std::isfinite(v[i])) return false; return true; };
    switch (r->kind) {
    case SIMLOD_REGION_BOX:
        if (!finite(r->box_min, 3) || !finite(r->box_max, 3)) return fail(SIMLOD_ERR_INVALID, "region box has a non-finite bound");
        for (int a = 0; a < 3; a++)
            if (r->box_min[a] > r->box_max[a]) return fail(SIMLOD_ERR_INVALID, "region box has min > max on axis %d", a);
        return SIMLOD_OK;
    case SIMLOD_REGION_SPHERE:
        if (!finite(r->center, 3) || !std::isfinite(r->radius)) return fail(SIMLOD_ERR_INVALID, "region sphere has a non-finite centre or radius");
        if (r->radius < 0.0f) return fail(SIMLOD_ERR_INVALID, "region sphere has a negative radius");
        return SIMLOD_OK;
    case SIMLOD_REGION_PLANES:
        if (r->num_planes == 0 || r->num_planes > SIMLOD_REGION_MAX_PLANES)
            return fail(SIMLOD_ERR_INVALID, "region has %u planes, 1 to %d are supported", r->num_planes, (int)SIMLOD_REGION_MAX_PLANES);
        if (!finite(&r->planes[0][0], 4 * (int)r->num_planes)) return fail(SIMLOD_ERR_INVALID, "region has a non-finite plane coefficient");
        return SIMLOD_OK;
    }
    return fail(SIMLOD_ERR_INVALID, "unknown region kind %u", r->kind);
}
}  // namespace

// ---- clip volumes (DESIGN.md §9.15): render.cu's simlod_render_clip and pick.cu apply the context's clip ------------------
int simlod_set_clip(SimlodContext* ctx, const SimlodClip* clip) {
    if (!ctx) return fail(SIMLOD_ERR_INVALID, "null context");
    if (!clip || clip->mode == SIMLOD_CLIP_NONE) { ctx->clip = SimlodClip{}; return SIMLOD_OK; }
    if (clip->mode != SIMLOD_CLIP_INSIDE && clip->mode != SIMLOD_CLIP_OUTSIDE) return fail(SIMLOD_ERR_INVALID, "unknown clip mode %u", clip->mode);
    if (clip->num_regions == 0 || clip->num_regions > SIMLOD_CLIP_MAX_REGIONS)
        return fail(SIMLOD_ERR_INVALID, "clip has %u regions, 1 to %d are supported", clip->num_regions, (int)SIMLOD_CLIP_MAX_REGIONS);
    for (uint32_t k = 0; k < clip->num_regions; k++) {
        int rc = checkRegion(&clip->regions[k]);
        if (rc) return fail(rc, "clip region %u: %s", k, g_error.c_str());
    }
    ctx->clip = *clip;
    return SIMLOD_OK;
}

int simlod_query_region(SimlodContext* ctx, const SimlodRegion* region, int32_t depth, uint64_t dst_samples,
                        uint64_t sample_capacity, SimlodQueryInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!info) return fail(SIMLOD_ERR_INVALID, "null info");
    rc = checkDepth("query", depth); if (rc) return rc;
    rc = checkAligned("query", {{"dst_samples", dst_samples, 16}}); if (rc) return rc;
    rc = checkRegion(region); if (rc) return rc;
    Scratch sc;
    rc = scratchFor(ctx, ScratchUse::QUERY, &sc); if (rc) return rc;
    CUdeviceptr nodes = ctx->buf.nodes, stats = ctx->buf.stats;
    SimlodRegion rg = *region;
    QueryBox box;
    std::copy_n(ctx->uniforms.boxMin, 3, box.mn); std::copy_n(ctx->uniforms.boxMax, 3, box.mx);
    // stage 1, into scratch only: plan (one block), the chunk-list walk, the per-item counts and their scan
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_QUERY_PLAN], 1, 1024, ctx->streamMain, nodes, stats, depth, sc.maxRecords, sc.rec, sc.recNode, sc.recItem, sc.ctl, rg, box);
    if (rc) return rc;
    rc = launchCollect(ctx, sc); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_QUERY_COUNT], (unsigned)ctx->numSMs * 8, 256, ctx->streamMain, sc.items, sc.rec, sc.recItem, sc.words, sc.ctl, rg, box);
    if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_QUERY_SCAN], 1, 1024, ctx->streamMain, sc.words, sc.ctl); if (rc) return rc;
    QueryCtl c;
    float ms = 0.0f;
    rc = clock.finish(&ms, {{sc.ctl, &c, sizeof c}}); if (rc) return rc;
    if (kernel_ms) *kernel_ms = ms;
    if (c.plan.error) return failInconsistent(c.plan.error);
    info->num_samples = c.outSamples; info->num_points = c.outPoints; info->num_voxels = c.outVoxels;
    info->samples_tested = c.plan.numSamples; info->nodes_visited = c.nodesVisited; info->max_level = c.plan.maxLevel;
    if (!dst_samples) return SIMLOD_OK;                         // size query
    if (sample_capacity < c.outSamples)
        return fail(SIMLOD_ERR_INVALID, "sample destination holds %llu samples, the query returns %llu", (unsigned long long)sample_capacity, (unsigned long long)c.outSamples);
    if (!c.outSamples) return SIMLOD_OK;
    // stage 2: the passing samples into the destination
    CUdeviceptr ds = (CUdeviceptr)dst_samples;
    StageClock write(ctx); rc = write.mark(); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_QUERY_WRITE], (unsigned)ctx->numSMs * 8, 256, ctx->streamMain, sc.items, sc.words, ds, sc.ctl, rg, box);
    if (rc) return rc;
    float writeMs = 0.0f;
    rc = write.finish(&writeMs); if (rc) return rc;
    if (kernel_ms) *kernel_ms = ms + writeMs;
    return SIMLOD_OK;
}

// ---- pick (DESIGN.md §9.9); kernels in pick.cu, the plan is the view export's ------------------------------------------
int simlod_pick(SimlodContext* ctx, const uint32_t* pixels, uint64_t num_pixels, uint64_t dst_index, uint64_t dst_samples,
                SimlodPickInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!info) return fail(SIMLOD_ERR_INVALID, "null info");
    const uint32_t width = ctx->cfg.width, height = ctx->cfg.height;
    const uint64_t frame = (uint64_t)width * height;
    std::vector<uint32_t> ids;
    if (pixels) {
        if (num_pixels == 0 || num_pixels > frame)
            return fail(SIMLOD_ERR_INVALID, "pixel list of %llu pixels, 1 to %llu (the frame) are supported", (unsigned long long)num_pixels, (unsigned long long)frame);
        ids.resize(num_pixels);
        for (uint64_t t = 0; t < num_pixels; t++) {
            const uint32_t x = pixels[2 * t], y = pixels[2 * t + 1];
            if (x >= width || y >= height)
                return fail(SIMLOD_ERR_INVALID, "pixel %llu (%u, %u) lies outside the %ux%u frame", (unsigned long long)t, x, y, width, height);
            ids[t] = x + width * y;
        }
    } else if (num_pixels) {
        return fail(SIMLOD_ERR_INVALID, "num_pixels without a pixel list");
    }
    rc = checkAligned("pick", {{"dst_index", dst_index, 8}, {"dst_samples", dst_samples, 16}}); if (rc) return rc;
    const uint32_t n = (uint32_t)(pixels ? num_pixels : frame);
    // stage 1: the view export's plan, into its scratch, and the one host round trip for its control word
    ExportPlanned p;
    rc = exportPlan(ctx, -1, &ctx->uniforms, &p, kernel_ms); if (rc) return rc;
    // stage 2: the two frames, then the indices of the requested pixels
    Layout l;
    const uint64_t oKey = l.take(8 * frame), oIndex = l.take(8 * frame), oHits = l.take(8), oList = l.take(4ull * n);
    rc = growDevice(&ctx->queryScratch, &ctx->queryScratchBytes, l.bytes); if (rc) return rc;
    const CUdeviceptr base = ctx->queryScratch, list = pixels ? base + oList : 0;
    if (pixels) CU(D(cuMemcpyHtoDAsync)(list, ids.data(), 4ull * n, ctx->streamMain));
    PickArgs a{devPtr(p.s.rec), devPtr(p.s.recItem), devPtr(p.s.items), devPtr(base + oKey), devPtr(base + oIndex), devPtr(base + oHits),
               p.c.numItems, p.c.numNodes, 0, ctx->clip};
    SimlodUniforms u = ctx->uniforms;
    CUdeviceptr di = (CUdeviceptr)dst_index, ds = (CUdeviceptr)dst_samples;
    uint32_t count = n;
    const unsigned blocks = (unsigned)ctx->numSMs * 4;
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_PICK_CLEAR], blocks, 256, ctx->streamMain, u, a); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_PICK_KEY], blocks, 256, ctx->streamMain, u, a); if (rc) return rc;
    rc = clock.mark(); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_PICK_INDEX], blocks, 256, ctx->streamMain, u, a); if (rc) return rc;
    rc = clock.mark(); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_PICK_WRITE], blocks, 256, ctx->streamMain, a, list, count, di, ds); if (rc) return rc;
    uint64_t hits = 0;
    float ms[3] = {};                                           // key, index, write
    rc = clock.finish(ms, {{base + oHits, &hits, sizeof hits}}); if (rc) return rc;
    info->num_hits = hits; info->num_samples = p.c.numSamples; info->num_nodes = p.c.numNodes; info->num_pixels = n;
    info->plan_ms = p.ms; info->key_ms = ms[0]; info->index_ms = ms[1]; info->write_ms = ms[2];
    if (kernel_ms) *kernel_ms = p.ms + ms[0] + ms[1] + ms[2];
    return SIMLOD_OK;
}

// ---- k nearest samples (DESIGN.md §9.10); kernels in nearest.cu, the plan is the export's -------------------------------
namespace {
// The queries bucketed by home record (nearest.cu's locate, scan and scatter), in the context's query scratch: per query
// home | slot | bucket, per home count | offset | run start, NearestCtl, then `extraBytes` for the caller at *extra.
// Fills the NearestArgs of the bucketing (no destinations) and enqueues its clears and three kernels.
int launchBuckets(SimlodContext* ctx, const ExportPlanned& p, uint64_t queries, uint32_t n, int32_t depth, uint64_t extraBytes,
                  NearestArgs* out, CUdeviceptr* extra) {
    const uint32_t homes = p.c.numNodes + 1;
    Layout l;
    const uint64_t oHome = l.take(4ull * n), oSlot = l.take(4ull * n), oBucket = l.take(4ull * n);
    const uint64_t oCount = l.take(4ull * homes), oOffset = l.take(4ull * homes), oRun = l.take(4ull * (homes + 1)), oCtl = l.take(sizeof(NearestCtl));
    const uint64_t oExtra = l.take(extraBytes);
    int rc = growDevice(&ctx->queryScratch, &ctx->queryScratchBytes, l.bytes); if (rc) return rc;
    const CUdeviceptr base = ctx->queryScratch;
    NearestArgs a = planArgs<NearestArgs>(p, ctx->uniforms, depth);
    a.queries = devPtr(queries);
    a.home = devPtr(base + oHome); a.slot = devPtr(base + oSlot); a.bucket = devPtr(base + oBucket);
    a.count = devPtr(base + oCount); a.offset = devPtr(base + oOffset); a.runStart = devPtr(base + oRun); a.ctl = devPtr(base + oCtl);
    a.numQueries = n; a.k = 1; a.maxRadius = INFINITY;
    *out = a;
    if (extra) *extra = base + oExtra;
    const unsigned blocks = (unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)ctx->numSMs * 8);
    CU(D(cuMemsetD32Async)(base + oCount, 0, homes, ctx->streamMain));
    CU(D(cuMemsetD8Async)(base + oCtl, 0, sizeof(NearestCtl), ctx->streamMain));
    rc = launch(ctx, ctx->fn[K_NEAREST_LOCATE], blocks, 256, ctx->streamMain, a); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_NEAREST_SCAN], 1, 1024, ctx->streamMain, a); if (rc) return rc;
    return launch(ctx, ctx->fn[K_NEAREST_SCATTER], blocks, 256, ctx->streamMain, a);
}

// The grid of a search over the buckets: the upper bound ceil(n / NEAREST_RUN) + min(n, homes) of the runs the scan
// counts; the blocks beyond return
unsigned searchRuns(uint32_t n, uint32_t records) {
    return (unsigned)((n + NEAREST_RUN - 1) / NEAREST_RUN + std::min<uint64_t>(n, (uint64_t)records + 1));
}
}  // namespace

int simlod_query_nearest(SimlodContext* ctx, uint64_t queries, uint64_t num_queries, uint32_t k, int32_t depth, float max_radius,
                         uint64_t dst_index, uint64_t dst_dist2, uint64_t dst_samples, SimlodNearestInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!info) return fail(SIMLOD_ERR_INVALID, "null info");
    if (k < 1 || k > SIMLOD_NEAREST_MAX_K) return fail(SIMLOD_ERR_INVALID, "k = %u, 1 to %d are supported", k, (int)SIMLOD_NEAREST_MAX_K);
    if (num_queries == 0 || num_queries > SIMLOD_NEAREST_MAX_QUERIES)
        return fail(SIMLOD_ERR_INVALID, "%llu queries, 1 to %u are supported", (unsigned long long)num_queries, (unsigned)SIMLOD_NEAREST_MAX_QUERIES);
    rc = checkDepth("nearest", depth); if (rc) return rc;
    if (std::isnan(max_radius) || max_radius < 0.0f) return fail(SIMLOD_ERR_INVALID, "max_radius must be >= 0 or +inf");
    rc = checkAligned("nearest", {{"queries", queries, 16, true}, {"dst_index", dst_index, 8}, {"dst_dist2", dst_dist2, 4}, {"dst_samples", dst_samples, 16}}); if (rc) return rc;
    const uint32_t n = (uint32_t)num_queries;
    // stage 1: the export's plan and chunk items, into its scratch, and the one host round trip for its control word
    ExportPlanned p;
    rc = exportPlan(ctx, depth < 0 ? -1 : depth, nullptr, &p, kernel_ms); if (rc) return rc;
    // stage 2: locate and bucket the queries; stage 3: the search, which writes the destinations unless the scan found
    // the record tree inconsistent
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    NearestArgs a{};
    rc = launchBuckets(ctx, p, queries, n, depth, 0, &a, nullptr); if (rc) return rc;
    a.dstIndex = devPtr(dst_index); a.dstDist2 = devPtr(dst_dist2); a.dstSamples = devPtr(dst_samples);
    a.k = k; a.maxRadius = max_radius;
    rc = clock.mark(); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_NEAREST_SEARCH], searchRuns(n, p.c.numNodes), NEAREST_RUN * 32, ctx->streamMain, a); if (rc) return rc;
    NearestCtl c;
    float ms[2] = {};                                           // bucket, search
    rc = clock.finish(ms, {{(CUdeviceptr)(uintptr_t)a.ctl, &c, sizeof c}}); if (rc) return rc;
    if (kernel_ms) *kernel_ms = p.ms + ms[0] + ms[1];
    if (c.error) return failInconsistent(c.error);
    *info = SimlodNearestInfo{};
    info->num_samples = p.c.numSamples; info->num_found = c.numFound; info->samples_tested = c.samplesTested;
    info->records_visited = c.recordsVisited; info->num_queries = n; info->k = k; info->invalid_queries = (uint32_t)c.invalid;
    info->max_level = p.c.maxLevel; info->plan_ms = p.ms; info->bucket_ms = ms[0]; info->search_ms = ms[1];
    return SIMLOD_OK;
}

// ---- fixed-radius neighbourhoods (DESIGN.md §9.12); kernels in radius.cu after nearest.cu's bucketing -------------------
int simlod_query_radius(SimlodContext* ctx, uint64_t queries, uint64_t num_queries, float radius, int32_t depth,
                        uint64_t dst_offsets, uint64_t dst_index, uint64_t dst_dist2, uint64_t dst_samples,
                        uint64_t capacity, SimlodRadiusInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!info) return fail(SIMLOD_ERR_INVALID, "null info");
    if (!std::isfinite(radius) || radius < 0.0f) return fail(SIMLOD_ERR_INVALID, "radius must be finite and >= 0");
    if (num_queries == 0 || num_queries > SIMLOD_RADIUS_MAX_QUERIES)
        return fail(SIMLOD_ERR_INVALID, "%llu queries, 1 to %u are supported", (unsigned long long)num_queries, (unsigned)SIMLOD_RADIUS_MAX_QUERIES);
    rc = checkDepth("radius", depth); if (rc) return rc;
    rc = checkAligned("radius", {{"queries", queries, 16, true}, {"dst_offsets", dst_offsets, 8}, {"dst_index", dst_index, 8},
                                 {"dst_dist2", dst_dist2, 4}, {"dst_samples", dst_samples, 16}}); if (rc) return rc;
    const uint32_t n = (uint32_t)num_queries;
    const bool sizeQuery = !dst_index && !dst_dist2 && !dst_samples;
    // stage 1: the export's plan and chunk items, into its scratch, and the one host round trip for its control word
    ExportPlanned p;
    rc = exportPlan(ctx, depth < 0 ? -1 : depth, nullptr, &p, kernel_ms); if (rc) return rc;
    // stage 2: locate and bucket the queries (nearest.cu); stage 3: count, reduce and scan, then one host round trip
    const uint32_t tiles = (n + RADIUS_SCAN_TILE - 1) / RADIUS_SCAN_TILE;
    Layout l;
    const uint64_t oCtl = l.take(sizeof(RadiusCtl)), oTotal = l.take(4ull * n), oBefore = l.take(4ull * n), oTile = l.take(8ull * tiles),
                   oOffsets = l.take(8ull * (n + 1));
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    NearestArgs na{};
    CUdeviceptr base = 0;
    rc = launchBuckets(ctx, p, queries, n, depth, l.bytes, &na, &base); if (rc) return rc;
    RadiusArgs a = planArgs<RadiusArgs>(p, ctx->uniforms, depth);
    a.queries = devPtr(queries);
    a.count = na.count; a.offset = na.offset; a.runStart = na.runStart; a.bucket = na.bucket; a.nearestCtl = na.ctl;
    a.ctl = devPtr(base + oCtl); a.total = devPtr(base + oTotal); a.before = devPtr(base + oBefore); a.tileSum = devPtr(base + oTile);
    a.offsets = devPtr(base + oOffsets);
    a.dstIndex = devPtr(dst_index); a.dstDist2 = devPtr(dst_dist2); a.dstSamples = devPtr(dst_samples);
    a.numQueries = n; a.radius = radius;
    CU(D(cuMemsetD8Async)(base + oCtl, 0, sizeof(RadiusCtl), ctx->streamMain));
    rc = clock.mark(); if (rc) return rc;
    const unsigned runs = searchRuns(n, p.c.numNodes);
    rc = launch(ctx, ctx->fn[K_RADIUS_COUNT], runs, NEAREST_RUN * 32, ctx->streamMain, a); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_RADIUS_REDUCE], tiles, 1024, ctx->streamMain, a); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_RADIUS_SCAN], tiles, 1024, ctx->streamMain, a); if (rc) return rc;
    NearestCtl nc;
    RadiusCtl c;
    float ms[2] = {};                                           // bucket, count
    rc = clock.finish(ms, {{(CUdeviceptr)(uintptr_t)na.ctl, &nc, sizeof nc}, {base + oCtl, &c, sizeof c}}); if (rc) return rc;
    if (kernel_ms) *kernel_ms = p.ms + ms[0] + ms[1];
    if (nc.error) return failInconsistent(nc.error);
    *info = SimlodRadiusInfo{};
    info->num_samples = p.c.numSamples; info->num_found = c.numFound; info->samples_tested = c.samplesTested;
    info->records_visited = c.recordsVisited; info->num_queries = n; info->invalid_queries = (uint32_t)c.invalid;
    info->max_level = p.c.maxLevel; info->max_found = c.maxFound;
    info->plan_ms = p.ms; info->bucket_ms = ms[0]; info->count_ms = ms[1];
    if (sizeQuery) {                                            // size query: the offsets at most
        if (dst_offsets) {
            CU(D(cuMemcpyDtoDAsync)((CUdeviceptr)dst_offsets, base + oOffsets, 8ull * (n + 1), ctx->streamMain));
            CU(D(cuStreamSynchronize)(ctx->streamMain));
        }
        return SIMLOD_OK;
    }
    if (capacity < c.numFound)
        return fail(SIMLOD_ERR_INVALID, "radius destinations hold %llu neighbours, the query finds %llu", (unsigned long long)capacity, (unsigned long long)c.numFound);
    // stage 4: the offsets, and the write pass, which places every neighbour
    StageClock write(ctx); rc = write.mark(); if (rc) return rc;
    if (dst_offsets) CU(D(cuMemcpyDtoDAsync)((CUdeviceptr)dst_offsets, base + oOffsets, 8ull * (n + 1), ctx->streamMain));
    rc = launch(ctx, ctx->fn[K_RADIUS_WRITE], runs, NEAREST_RUN * 32, ctx->streamMain, a); if (rc) return rc;
    float writeMs = 0.0f;
    rc = write.finish(&writeMs); if (rc) return rc;
    info->write_ms = writeMs;
    if (kernel_ms) *kernel_ms = p.ms + ms[0] + ms[1] + writeMs;
    return SIMLOD_OK;
}

// ---- rays (DESIGN.md §9.11); kernels in ray.cu, the plan is the export's ------------------------------------------------
int simlod_query_ray(SimlodContext* ctx, uint64_t rays, uint64_t num_rays, float radius, int32_t depth, uint64_t dst_index,
                     uint64_t dst_t, uint64_t dst_h2, uint64_t dst_samples, SimlodRayInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!info) return fail(SIMLOD_ERR_INVALID, "null info");
    if (!std::isfinite(radius) || radius < 0.0f) return fail(SIMLOD_ERR_INVALID, "radius must be finite and >= 0");
    if (num_rays == 0 || num_rays > SIMLOD_RAY_MAX_RAYS)
        return fail(SIMLOD_ERR_INVALID, "%llu rays, 1 to %u are supported", (unsigned long long)num_rays, (unsigned)SIMLOD_RAY_MAX_RAYS);
    rc = checkDepth("ray", depth); if (rc) return rc;
    rc = checkAligned("ray", {{"rays", rays, 16, true}, {"dst_index", dst_index, 8}, {"dst_t", dst_t, 4}, {"dst_h2", dst_h2, 4},
                              {"dst_samples", dst_samples, 16}}); if (rc) return rc;
    const uint32_t n = (uint32_t)num_rays;
    // stage 1: the export's plan and chunk items, into its scratch, and the one host round trip for its control word
    ExportPlanned p;
    rc = exportPlan(ctx, depth < 0 ? -1 : depth, nullptr, &p, kernel_ms); if (rc) return rc;
    rc = growDevice(&ctx->queryScratch, &ctx->queryScratchBytes, sizeof(RayCtl)); if (rc) return rc;
    RayArgs a = planArgs<RayArgs>(p, ctx->uniforms, depth);
    a.rays = devPtr(rays); a.ctl = devPtr(ctx->queryScratch);
    a.dstIndex = devPtr(dst_index); a.dstT = devPtr(dst_t); a.dstH2 = devPtr(dst_h2); a.dstSamples = devPtr(dst_samples);
    a.numRays = n; a.radius = radius;
    // stage 2: the level check, then the trace, which writes the destinations unless the check found the record tree
    // inconsistent
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    CU(D(cuMemsetD8Async)(ctx->queryScratch, 0, sizeof(RayCtl), ctx->streamMain));
    rc = launch(ctx, ctx->fn[K_RAY_CHECK], 1, 1024, ctx->streamMain, a); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_RAY_TRACE], (n + RAY_WARPS - 1) / RAY_WARPS, RAY_WARPS * 32, ctx->streamMain, a); if (rc) return rc;
    RayCtl c;
    float traceMs = 0.0f;
    rc = clock.finish(&traceMs, {{ctx->queryScratch, &c, sizeof c}}); if (rc) return rc;
    if (kernel_ms) *kernel_ms = p.ms + traceMs;
    if (c.error) return failInconsistent(c.error);
    *info = SimlodRayInfo{};
    info->num_samples = p.c.numSamples; info->num_hits = c.numHits; info->samples_tested = c.samplesTested;
    info->records_visited = c.recordsVisited; info->num_rays = n; info->invalid_rays = (uint32_t)c.invalid;
    info->max_level = p.c.maxLevel; info->plan_ms = p.ms; info->trace_ms = traceMs;
    return SIMLOD_OK;
}

// ---- height maps (DESIGN.md §9.14); kernels in heightmap.cu, the plan is the export's -----------------------------------
int simlod_query_heightmap(SimlodContext* ctx, const SimlodHeightmap* grid, int32_t depth, uint64_t dst_count, uint64_t dst_z_min,
                           uint64_t dst_z_max, uint64_t dst_z_mean, uint64_t dst_top, uint64_t dst_samples,
                           SimlodHeightmapInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!info) return fail(SIMLOD_ERR_INVALID, "null info");
    if (!grid) return fail(SIMLOD_ERR_INVALID, "null grid");
    const SimlodHeightmap g = *grid;
    if (!std::isfinite(g.origin[0]) || !std::isfinite(g.origin[1])) return fail(SIMLOD_ERR_INVALID, "heightmap origin must be finite");
    if (!std::isfinite(g.cell) || !(g.cell > 0.0f)) return fail(SIMLOD_ERR_INVALID, "heightmap cell must be finite and > 0");
    const uint64_t cells = (uint64_t)g.nx * g.ny;
    if (cells == 0 || cells > SIMLOD_HEIGHTMAP_MAX_CELLS)
        return fail(SIMLOD_ERR_INVALID, "heightmap of %u x %u cells, 1 to %u cells are supported (tile larger rasters)", g.nx, g.ny,
                    (unsigned)SIMLOD_HEIGHTMAP_MAX_CELLS);
    rc = checkDepth("heightmap", depth); if (rc) return rc;
    rc = checkAligned("heightmap", {{"dst_count", dst_count, 8}, {"dst_z_min", dst_z_min, 4}, {"dst_z_max", dst_z_max, 4},
                                    {"dst_z_mean", dst_z_mean, 4}, {"dst_top", dst_top, 8}, {"dst_samples", dst_samples, 16}}); if (rc) return rc;
    // stage 1: the export's plan and chunk items, into its scratch, and the one host round trip for its control word
    ExportPlanned p;
    rc = exportPlan(ctx, depth < 0 ? -1 : depth, nullptr, &p, kernel_ms); if (rc) return rc;
    if (p.c.numSamples >> 32)
        return fail(SIMLOD_ERR_INVALID, "heightmap: the export holds %llu samples, at most 2^32 - 1 are supported", (unsigned long long)p.c.numSamples);
    // the accumulators a destination needs; the count is always kept, for the info
    const bool wantMin = dst_z_min, wantTop = dst_z_max || dst_top || dst_samples, wantSum = dst_z_mean;
    Layout l;
    const uint64_t oCtl = l.take(sizeof(HeightmapCtl)), oCount = l.take(4 * cells), oMin = l.take(wantMin ? 4 * cells : 0),
                   oTop = l.take(wantTop ? 8 * cells : 0), oSum = l.take(wantSum ? 8 * cells : 0);
    rc = growDevice(&ctx->queryScratch, &ctx->queryScratchBytes, l.bytes); if (rc) return rc;
    const CUdeviceptr base = ctx->queryScratch;
    HeightmapArgs a = planArgs<HeightmapArgs>(p, ctx->uniforms, depth);
    a.ctl = devPtr(base + oCtl); a.count = devPtr(base + oCount);
    a.zmin = devPtr(wantMin ? base + oMin : 0); a.top = devPtr(wantTop ? base + oTop : 0); a.sum = devPtr(wantSum ? base + oSum : 0);
    a.dstCount = devPtr(dst_count); a.dstZMin = devPtr(dst_z_min); a.dstZMax = devPtr(dst_z_max); a.dstZMean = devPtr(dst_z_mean);
    a.dstTop = devPtr(dst_top); a.dstSamples = devPtr(dst_samples);
    a.numItems = p.c.numItems; a.nx = g.nx; a.ny = g.ny;
    a.origin[0] = g.origin[0]; a.origin[1] = g.origin[1]; a.cell = g.cell;
    // stage 2: reset the accumulators (memsets) and bin every sample; stage 3: the destinations
    StageClock clock(ctx); rc = clock.mark(); if (rc) return rc;
    CU(D(cuMemsetD8Async)(base + oCtl, 0, sizeof(HeightmapCtl), ctx->streamMain));
    CU(D(cuMemsetD32Async)(base + oCount, 0, cells, ctx->streamMain));
    if (wantMin) CU(D(cuMemsetD32Async)(base + oMin, 0xffffffffu, cells, ctx->streamMain));
    if (wantTop) CU(D(cuMemsetD8Async)(base + oTop, 0, 8 * cells, ctx->streamMain));
    if (wantSum) CU(D(cuMemsetD8Async)(base + oSum, 0, 8 * cells, ctx->streamMain));
    rc = launch(ctx, ctx->fn[K_HEIGHTMAP_ACCUMULATE], (unsigned)ctx->numSMs * 8, 256, ctx->streamMain, a); if (rc) return rc;
    rc = clock.mark(); if (rc) return rc;
    const unsigned blocks = (unsigned)std::min<uint64_t>((cells + 255) / 256, (uint64_t)ctx->numSMs * 8);
    rc = launch(ctx, ctx->fn[K_HEIGHTMAP_FINALIZE], blocks, 256, ctx->streamMain, a); if (rc) return rc;
    HeightmapCtl c;
    float ms[2] = {};                                           // reset + accumulate, finalize
    rc = clock.finish(ms, {{base + oCtl, &c, sizeof c}}); if (rc) return rc;
    if (kernel_ms) *kernel_ms = p.ms + ms[0] + ms[1];
    *info = SimlodHeightmapInfo{};
    info->num_samples = p.c.numSamples; info->num_binned = c.numBinned; info->samples_tested = c.samplesTested;
    info->records_visited = c.recordsVisited; info->nonempty_cells = c.nonemptyCells; info->max_level = p.c.maxLevel;
    info->plan_ms = p.ms; info->accumulate_ms = ms[0]; info->finalize_ms = ms[1];
    return SIMLOD_OK;
}

// ---- octree files (DESIGN.md §9.7); kernels in export.cu (save) and import.cu (load) ---------------------------------
}  // extern "C"

namespace {
constexpr uint64_t FILE_WINDOW_BYTES = POOL_BYTES / 2;             // samples per staged window: half the page-locked pool
constexpr uint64_t FILE_WINDOW_SAMPLES = FILE_WINDOW_BYTES / sizeof(SimlodPoint);
constexpr uint32_t NODE_TABLE_CAP = (uint32_t)scratch::NODE_CAP;  // the builder's side tables
constexpr uint32_t ROW_CAP = (uint32_t)scratch::ROW_CAP, ROW_SLOTS = (uint32_t)scratch::ROW_SLOTS;   // chunk rows

// where each section of a file with n records and s samples lies (SimlodOctreeFileHeader)
void octreeLayout(uint64_t n, uint64_t s, SimlodOctreeFileHeader* h) {
    h->records_offset = SIMLOD_OCTREE_HEADER_SIZE;
    h->counters_offset = h->records_offset + n * sizeof(SimlodExportNode);
    h->samples_offset = align16(h->counters_offset + 4 * n);
    h->file_size = h->samples_offset + s * sizeof(SimlodPoint);
}

int readOctreeHeader(const char* path, SimlodOctreeFileHeader* out) {
    struct stat st;
    if (stat(path, &st) != 0) return fail(SIMLOD_ERR_INVALID, "cannot open %s", path);
    FILE* f = fopen(path, "rb");
    if (!f) return fail(SIMLOD_ERR_INVALID, "cannot open %s", path);
    SimlodOctreeFileHeader h;
    const size_t got = fread(&h, 1, sizeof(h), f);
    fclose(f);
    if (got != sizeof(h)) return fail(SIMLOD_ERR_INVALID, "%s is shorter than an octree file header (%zu bytes)", path, got);
    if (memcmp(h.magic, SIMLOD_OCTREE_MAGIC, 8) != 0) return fail(SIMLOD_ERR_INVALID, "%s is not an octree file (no SIMLODOT magic)", path);
    if (h.version != SIMLOD_OCTREE_VERSION) return fail(SIMLOD_ERR_INVALID, "%s: octree file version %u, this library reads version %d", path, h.version, (int)SIMLOD_OCTREE_VERSION);
    if (h.header_size != SIMLOD_OCTREE_HEADER_SIZE) return fail(SIMLOD_ERR_INVALID, "%s: header size %u, expected %d", path, h.header_size, (int)SIMLOD_OCTREE_HEADER_SIZE);
    if (h.info.num_nodes == 0 || h.info.num_points + h.info.num_voxels != h.info.num_samples || h.info.num_samples < h.info.num_points ||
        h.info.num_samples > (std::numeric_limits<uint64_t>::max() >> 5) || h.info.max_level > SIMLOD_MAX_DEPTH || h.reserved0 || h.reserved1)
        return fail(SIMLOD_ERR_INVALID, "%s: inconsistent header (%u records, %llu samples = %llu points + %llu voxels, deepest level %u)", path,
                    h.info.num_nodes, (unsigned long long)h.info.num_samples, (unsigned long long)h.info.num_points, (unsigned long long)h.info.num_voxels, h.info.max_level);
    SimlodOctreeFileHeader want = h;
    octreeLayout(h.info.num_nodes, h.info.num_samples, &want);
    if (h.records_offset != want.records_offset || h.counters_offset != want.counters_offset || h.samples_offset != want.samples_offset ||
        h.file_size != want.file_size)
        return fail(SIMLOD_ERR_INVALID, "%s: section offsets (%llu, %llu, %llu, size %llu) disagree with %u records and %llu samples", path,
                    (unsigned long long)h.records_offset, (unsigned long long)h.counters_offset, (unsigned long long)h.samples_offset,
                    (unsigned long long)h.file_size, h.info.num_nodes, (unsigned long long)h.info.num_samples);
    if ((uint64_t)st.st_size != h.file_size)
        return fail(SIMLOD_ERR_INVALID, "%s is %llu bytes, its header describes %llu", path, (unsigned long long)st.st_size, (unsigned long long)h.file_size);
    *out = h;
    return SIMLOD_OK;
}

int ensureFileWindow(SimlodContext* ctx) {
    if (!ctx->fileWindow) CU(D(cuMemAlloc)(&ctx->fileWindow, FILE_WINDOW_BYTES));
    return ensurePinnedPool(ctx);
}

bool writeAll(FILE* f, const void* p, uint64_t bytes) { return bytes == 0 || fwrite(p, 1, bytes, f) == bytes; }

int saveOctree(SimlodContext* ctx, const char* path, SimlodExportInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!path) return fail(SIMLOD_ERR_INVALID, "null path");
    // the octree as the last completed launch left it
    CU(D(cuStreamSynchronize)(ctx->streamCopy));
    CU(D(cuStreamSynchronize)(ctx->streamUpload));
    rc = readStats(ctx); if (rc) return rc;
    const SimlodStats st = *ctx->hStats;
    if (st.dbg & ~(uint32_t)SIMLOD_DBG_FAR_POINT)
        return fail(SIMLOD_ERR_INVALID, "%s: not saved, the octree's Stats::dbg is 0x%x (a capacity of the builder was exceeded)", path, st.dbg);
    ExportPlanned p;
    rc = exportPlan(ctx, -1, nullptr, &p);
    if (rc) return fail(rc, "%s: not saved: %s", path, g_error.c_str());
    rc = ensureFileWindow(ctx); if (rc) return rc;
    float ms = p.ms;
    const uint32_t n = p.c.numNodes;
    const uint64_t numSamples = p.c.numSamples;
    SimlodOctreeFileHeader h;
    memset(&h, 0, sizeof(h));
    memcpy(h.magic, SIMLOD_OCTREE_MAGIC, 8);
    h.version = SIMLOD_OCTREE_VERSION;
    h.header_size = SIMLOD_OCTREE_HEADER_SIZE;
    h.info.num_nodes = n; h.info.max_level = p.c.maxLevel;
    h.info.num_samples = numSamples; h.info.num_points = p.c.numPoints; h.info.num_voxels = p.c.numVoxels;
    for (int i = 0; i < 3; i++) { h.box_min[i] = ctx->uniforms.boxMin[i]; h.box_max[i] = ctx->uniforms.boxMax[i]; }
    h.batchlet_index = st.batchletIndex;
    h.num_points_processed = st.numPointsProcessed;
    octreeLayout(n, numSamples, &h);
    // records and counters: bounded by nodes[]
    std::vector<uint8_t> head(h.samples_offset, 0);
    memcpy(head.data(), &h, sizeof(h));
    CU(D(cuMemcpyDtoH)(head.data() + h.records_offset, p.s.rec, (size_t)n * sizeof(SimlodExportNode)));
    CUdeviceptr nodes = ctx->buf.nodes, window = ctx->fileWindow;
    SimlodContext::LaunchQueue& q = ctx->queue;
    CU(D(cuEventRecord)(q.ev[0][0], ctx->streamMain));
    rc = launch(ctx, ctx->fn[K_EXPORT_COUNTERS], (unsigned)ctx->numSMs * 2, 256, ctx->streamMain, nodes, p.s.recNode, p.s.ctl, window);
    if (rc) return rc;
    CU(D(cuEventRecord)(q.ev[0][1], ctx->streamMain));
    CU(D(cuMemcpyDtoHAsync)(head.data() + h.counters_offset, window, (size_t)n * 4, ctx->streamMain));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    float t = 0.0f;
    CU(D(cuEventElapsedTime)(&t, q.ev[0][0], q.ev[0][1]));
    ms += t;
    // written under a temporary name and renamed once complete: a failed save leaves no partial file and replaces
    // no existing one
    const std::string tmpPath = std::string(path) + ".tmp";
    FILE* f = fopen(tmpPath.c_str(), "wb");
    if (!f) return fail(SIMLOD_ERR_INVALID, "cannot write %s", path);
    struct Closer {
        FILE*& f; const std::string& tmp; bool done = false;
        ~Closer() { if (f) fclose(f); if (!done) unlink(tmp.c_str()); }
    } closer{f, tmpPath};
    if (!writeAll(f, head.data(), head.size())) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);
    // samples: window w is gathered on the device and copied into pool half w & 1 while window w - 1 is written out
    const uint64_t numWindows = (numSamples + FILE_WINDOW_SAMPLES - 1) / FILE_WINDOW_SAMPLES;
    auto half = [&](uint64_t w) { return (char*)ctx->pinnedPool + (w & 1) * FILE_WINDOW_BYTES; };
    auto windowSamples = [&](uint64_t w) { return std::min<uint64_t>(FILE_WINDOW_SAMPLES, numSamples - w * FILE_WINDOW_SAMPLES); };
    auto drain = [&](uint64_t w) -> int {            // window w has been copied out: time it and write it
        CU(D(cuEventSynchronize)(q.statsDone[w & 1]));
        float g = 0.0f;
        CU(D(cuEventElapsedTime)(&g, q.ev[w & 1][0], q.ev[w & 1][1]));
        ms += g;
        if (!writeAll(f, half(w), windowSamples(w) * sizeof(SimlodPoint))) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);
        return SIMLOD_OK;
    };
    for (uint64_t w = 0; w < numWindows; w++) {
        uint64_t a = w * FILE_WINDOW_SAMPLES, b = a + windowSamples(w);
        CU(D(cuEventRecord)(q.ev[w & 1][0], ctx->streamMain));
        rc = launch(ctx, ctx->fn[K_EXPORT_GATHER_WINDOW], (unsigned)ctx->numSMs * 4, 256, ctx->streamMain, p.s.items, window, p.s.ctl, a, b);
        if (rc) return rc;
        CU(D(cuEventRecord)(q.ev[w & 1][1], ctx->streamMain));
        CU(D(cuMemcpyDtoHAsync)(half(w), window, (size_t)(b - a) * sizeof(SimlodPoint), ctx->streamMain));
        CU(D(cuEventRecord)(q.statsDone[w & 1], ctx->streamMain));
        if (w > 0) { rc = drain(w - 1); if (rc) return rc; }
    }
    if (numWindows > 0) { rc = drain(numWindows - 1); if (rc) return rc; }
    const int closed = fclose(f);
    f = nullptr;
    if (closed != 0) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);
    if (rename(tmpPath.c_str(), path) != 0) return fail(SIMLOD_ERR_INVALID, "cannot write %s (rename from %s failed)", path, tmpPath.c_str());
    closer.done = true;
    if (info) *info = h.info;
    if (kernel_ms) *kernel_ms = ms;
    return SIMLOD_OK;
}

// What load needs to know about a file's records beyond the records themselves: the heap plan and the Stats sweep.
struct LoadPlan {
    std::vector<ImportPlan> plan;      // one per record, then one with chunk = the total
    uint64_t gridBase = 0, chunkBase = 0, heapEnd = 0, numChunks = 0;
    uint32_t numGrids = 0, numRows = 0;
    SimlodStats stats{};               // the sweep fields
};

// The checks that make the records a full export of a builder's octree (simlod_load_octree), and the heap plan.
int planLoad(const char* path, const SimlodOctreeFileHeader& h, const SimlodExportNode* rec, const uint32_t* counters, LoadPlan* out) {
    const uint32_t n = h.info.num_nodes;
    auto bad = [&](uint32_t i, const char* what) { return fail(SIMLOD_ERR_INVALID, "%s: record %u: %s (not a full export of an octree)", path, i, what); };
    std::vector<ImportPlan>& plan = out->plan;
    plan.assign((size_t)n + 1, ImportPlan{0, 0, 0, 0});
    static const uint8_t rootName[20] = {'r'};
    if (rec[0].level != 0 || rec[0].X || rec[0].Y || rec[0].Z || rec[0].parent != -1 || memcmp(rec[0].name, rootName, 20) != 0) return bad(0, "not the root");
    uint32_t next = 1, maxLevel = 0, innerNonRoot = 0;
    uint64_t samples = 0, points = 0, voxels = 0, chunks = 0;
    SimlodStats& s = out->stats;
    for (uint32_t i = 0; i < n; i++) {
        const SimlodExportNode& r = rec[i];
        const bool inner = r.first_child >= 0;
        if (r.level > SIMLOD_MAX_DEPTH) return bad(i, "level above 20");
        if (r.first_child < -1) return bad(i, "bad first_child");
        if (r.flags != ((uint32_t)SIMLOD_EXPORT_SAMPLED | (inner ? 0u : (uint32_t)SIMLOD_EXPORT_LEAF))) return bad(i, "flags other than SAMPLED, and LEAF exactly on childless records");
        if (r.sample_offset != samples) return bad(i, "sample_offset is not the running sum");
        if (inner && r.num_points) return bad(i, "points on an inner node");
        if (!inner && i != 0 && r.num_voxels) return bad(i, "voxels on a leaf other than the root");
        if (!inner && counters[i] != r.num_points) return bad(i, "a leaf's counter differs from its point count");
        if (inner && counters[i] <= SIMLOD_MAX_POINTS_PER_NODE) return bad(i, "an inner node's counter is not above 50 000");
        if (!inner && r.level < SIMLOD_MAX_DEPTH && r.num_points > SIMLOD_MAX_POINTS_PER_NODE) return bad(i, "a leaf above level 20 holds more than 50 000 points");
        if (inner) {
            // children: the next 8 records, in child-index order, one level down (breadth-first order follows)
            if ((uint32_t)r.first_child != next || (uint64_t)next + 8 > n) return bad(i, "first_child is not the next 8 records in breadth-first order");
            for (uint32_t k = 0; k < 8; k++) {
                const SimlodExportNode& c = rec[next + k];
                uint8_t name[20];
                memcpy(name, r.name, 20);
                if (r.level + 1 < 20) name[r.level + 1] = (uint8_t)('0' + k);
                if (c.parent != (int32_t)i || c.level != r.level + 1 || c.X != 2 * r.X + ((k >> 2) & 1) || c.Y != 2 * r.Y + ((k >> 1) & 1) ||
                    c.Z != 2 * r.Z + (k & 1) || memcmp(c.name, name, 20) != 0)
                    return bad(next + k, "not the child of its parent (parent, level, X, Y, Z or name)");
            }
            next += 8;
            s.numInner++;
            s.numVoxels += r.num_voxels;
            s.numChunksVoxels += (r.num_voxels + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
        } else {
            s.numLeaves++;
            s.numPoints += r.num_points;
            s.numChunksPoints += (r.num_points + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
            if (r.num_points) s.numNonemptyLeaves++;
        }
        maxLevel = std::max(maxLevel, r.level);
        samples += (uint64_t)r.num_points + r.num_voxels;
        points += r.num_points;
        voxels += r.num_voxels;
        const uint32_t npc = (r.num_points + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
        if (npc > ROW_SLOTS) return fail(SIMLOD_ERR_CAPACITY, "%s: record %u holds %u point chunks, a leaf's chunk row holds %u", path, i, npc, ROW_SLOTS);
        plan[i].chunk = chunks;
        plan[i].counter = counters[i];
        plan[i].row = npc ? ++out->numRows : 0;
        plan[i].grid = i == 0 ? 16 : inner ? ++innerNonRoot : 0;        // grid index for now, offset below
        chunks += npc + (r.num_voxels + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
    }
    if (next != n) return bad(next < n ? next : n - 1, "records that no parent reaches");
    if (maxLevel != h.info.max_level || samples != h.info.num_samples || points != h.info.num_points || voxels != h.info.num_voxels)
        return fail(SIMLOD_ERR_INVALID, "%s: the records' counts disagree with the header", path);
    if (out->numRows > ROW_CAP) return fail(SIMLOD_ERR_CAPACITY, "%s: %u leaves hold points, the builder's chunk rows hold %u", path, out->numRows, ROW_CAP);
    out->gridBase = 16 + SIMLOD_GRID_STRIDE;
    out->chunkBase = out->gridBase + (uint64_t)innerNonRoot * SIMLOD_GRID_STRIDE;
    out->heapEnd = out->chunkBase + chunks * SIMLOD_CHUNK_STRIDE;
    out->numChunks = chunks;
    out->numGrids = innerNonRoot;
    for (uint32_t i = 1; i < n; i++) if (plan[i].grid) plan[i].grid = out->gridBase + (plan[i].grid - 1) * SIMLOD_GRID_STRIDE;
    plan[n].chunk = chunks;
    s.numNodes = n;
    s.numAllocatedChunks = s.chunkPoolSize = s.numChunksPoints;     // every point chunk in use, none free
    s.allocatedBytes_persistent = out->heapEnd;
    s.batchletIndex = h.batchlet_index;
    s.numPointsProcessed = h.num_points_processed;
    return SIMLOD_OK;
}

// chunk of the plan that holds sample `x` (x < total samples)
uint64_t chunkOfSample(const SimlodExportNode* rec, const std::vector<ImportPlan>& plan, uint32_t n, uint64_t x) {
    uint32_t lo = 0, hi = n;                                          // the last record whose sample_offset <= x
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) / 2; if (rec[mid].sample_offset <= x) lo = mid; else hi = mid; }
    const uint64_t local = x - rec[lo].sample_offset;
    const uint32_t np = rec[lo].num_points, npc = (np + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
    return plan[lo].chunk + (local < np ? local / SIMLOD_POINTS_PER_CHUNK : npc + (local - np) / SIMLOD_POINTS_PER_CHUNK);
}

bool preadAll(int fd, char* dst, uint64_t bytes, uint64_t at) {
    while (bytes) {
        const ssize_t r = pread(fd, dst, bytes, (off_t)at);
        if (r <= 0) return false;
        dst += r; at += (uint64_t)r; bytes -= (uint64_t)r;
    }
    return true;
}

int loadOctree(SimlodContext* ctx, const char* path, int loader_threads, SimlodExportInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!path) return fail(SIMLOD_ERR_INVALID, "null path");
    if (!ctx->programs[SIMLOD_PROGRAM_CONSTRUCT].builtin)
        return fail(SIMLOD_ERR_MODULE, "%s: not loaded, the builder's side tables are those of the built-in construct program and another one is in use", path);
    // ---- everything that can be refused is found before the context is written -------------------------------------
    SimlodOctreeFileHeader h;
    rc = readOctreeHeader(path, &h); if (rc) return rc;
    const uint32_t n = h.info.num_nodes;
    const uint32_t maxRecords = (uint32_t)std::min<uint64_t>(ctx->buf.nodes_bytes / sizeof(SimlodNode), NODE_TABLE_CAP);
    if (n > maxRecords) return fail(SIMLOD_ERR_CAPACITY, "%s holds %u nodes, nodes[] holds %u", path, n, maxRecords);
    int fd = open(path, O_RDONLY);
    if (fd < 0) return fail(SIMLOD_ERR_INVALID, "cannot open %s", path);
    struct FdCloser { int fd; ~FdCloser() { close(fd); } } fdCloser{fd};
    std::vector<uint8_t> head(h.samples_offset);
    if (!preadAll(fd, (char*)head.data(), head.size(), 0)) return fail(SIMLOD_ERR_INVALID, "read error in %s", path);
    const SimlodExportNode* rec = (const SimlodExportNode*)(head.data() + h.records_offset);
    const uint32_t* counters = (const uint32_t*)(head.data() + h.counters_offset);
    LoadPlan lp;
    rc = planLoad(path, h, rec, counters, &lp); if (rc) return rc;
    if (lp.heapEnd + HEAP_GUARD_BYTES >= ctx->buf.persistent_bytes)
        return fail(SIMLOD_ERR_CAPACITY, "%s needs %llu heap bytes, the persistent buffer holds %llu of which the capacity guard keeps the last %llu free", path,
                    (unsigned long long)lp.heapEnd, (unsigned long long)ctx->buf.persistent_bytes, (unsigned long long)HEAP_GUARD_BYTES);
    const uint64_t tableBytes = align16((uint64_t)maxRecords * sizeof(SimlodExportNode)) + align16((uint64_t)(maxRecords + 1) * sizeof(ImportPlan)) + 16;
    rc = growDevice(&ctx->fileTables, &ctx->fileTablesBytes, tableBytes); if (rc) return rc;
    rc = ensureFileWindow(ctx); if (rc) return rc;

    // ---- the context's octree is replaced from here on ------------------------------------------------------------------
    CU(D(cuStreamSynchronize)(ctx->streamCopy));
    CU(D(cuStreamSynchronize)(ctx->streamUpload));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    for (int i = 0; i < 3; i++) { ctx->uniforms.boxMin[i] = h.box_min[i]; ctx->uniforms.boxMax[i] = h.box_max[i]; }
    const CUdeviceptr recDev = ctx->fileTables, planDev = recDev + align16((uint64_t)maxRecords * sizeof(SimlodExportNode)),
                      errorDev = planDev + align16((uint64_t)(maxRecords + 1) * sizeof(ImportPlan));
    ImportArgs a{};
    a.nodes = devPtr(ctx->buf.nodes); a.heap = devPtr(ctx->buf.persistent); a.scratch = devPtr(ctx->buf.momentary);
    a.rec = devPtr(recDev); a.plan = devPtr(planDev); a.error = devPtr(errorDev);
    a.chunkBase = lp.chunkBase; a.numRecords = n; a.numRows = lp.numRows;
    for (int i = 0; i < 3; i++) { a.boxMin[i] = h.box_min[i]; a.boxMax[i] = h.box_max[i]; }
    const SimlodHeapHeader heapHeader{(uint8_t*)(uintptr_t)ctx->buf.persistent, lp.heapEnd};
    CU(D(cuMemsetD8Async)(ctx->buf.nodes, 0, ctx->buf.nodes_bytes, ctx->streamMain));
    CU(D(cuMemcpyHtoDAsync)(recDev, rec, (size_t)n * sizeof(SimlodExportNode), ctx->streamMain));
    CU(D(cuMemcpyHtoDAsync)(planDev, lp.plan.data(), lp.plan.size() * sizeof(ImportPlan), ctx->streamMain));
    CU(D(cuMemsetD32Async)(errorDev, 0, 1, ctx->streamMain));
    CU(D(cuMemcpyHtoDAsync)(ctx->buf.persistent, &heapHeader, sizeof(heapHeader), ctx->streamMain));
    CU(D(cuEventRecord)(ctx->evStart, ctx->streamMain));
    const unsigned blocks = (unsigned)ctx->numSMs * 4;
    uint64_t numChunks = lp.numChunks, gridBase = lp.gridBase;
    uint32_t numGrids = lp.numGrids;
    CUdeviceptr heap = ctx->buf.persistent;
    rc = launch(ctx, ctx->fn[K_IMPORT_NODES], blocks, 256, ctx->streamMain, a); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_IMPORT_LINK], blocks, 256, ctx->streamMain, a, numChunks); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_IMPORT_CLEAR_GRIDS], blocks * 2, 256, ctx->streamMain, heap, gridBase, numGrids); if (rc) return rc;
    CU(D(cuEventRecord)(ctx->evEnd, ctx->streamMain));
    // samples: loader threads read window w into pool half w & 1 while window w - 1 is copied and scattered
    const uint64_t numSamples = h.info.num_samples;
    const uint64_t numWindows = (numSamples + FILE_WINDOW_SAMPLES - 1) / FILE_WINDOW_SAMPLES;
    SimlodContext::LaunchQueue& q = ctx->queue;
    float ms = 0.0f, t = 0.0f;
    const int nThreads = std::max(1, std::min(loader_threads, 64));
    if (!ctx->loaderPool) ctx->loaderPool = new LoaderPool();
    LoaderPool* pool = ctx->loaderPool;
    bool readFailed = false;
    auto retire = [&](uint64_t w) -> int {           // the scatter of window w (and the copy before it) has completed
        CU(D(cuEventSynchronize)(q.ev[w & 1][1]));
        float g = 0.0f;
        CU(D(cuEventElapsedTime)(&g, q.ev[w & 1][0], q.ev[w & 1][1]));
        ms += g;
        return SIMLOD_OK;
    };
    for (uint64_t w = 0; w < numWindows && !readFailed; w++) {
        const uint64_t first = w * FILE_WINDOW_SAMPLES, count = std::min<uint64_t>(FILE_WINDOW_SAMPLES, numSamples - first);
        char* dst = (char*)ctx->pinnedPool + (w & 1) * FILE_WINDOW_BYTES;
        if (w >= 2) { rc = retire(w - 2); if (rc) return rc; }
        const uint64_t bytes = count * sizeof(SimlodPoint), at = h.samples_offset + first * sizeof(SimlodPoint);
        const uint64_t pieces = (bytes + PIECE_BYTES - 1) / PIECE_BYTES;
        std::atomic<uint64_t> nextPiece{0};
        std::atomic<bool> ok{true};
        pool->run(nThreads, [&, pool](int worker) {
            char* stage = pool->bounce[worker];
            for (uint64_t piece; (piece = nextPiece.fetch_add(1)) < pieces && ok.load();) {
                const uint64_t p0 = piece * PIECE_BYTES, pn = std::min<uint64_t>(PIECE_BYTES, bytes - p0);
                for (uint64_t done = 0; done < pn;) {
                    const uint64_t want = std::min<uint64_t>(pn - done, LoaderPool::BOUNCE_BYTES);
                    if (!preadAll(fd, stage, want, at + p0 + done)) { ok.store(false); break; }
                    copyStreaming(dst + p0 + done, stage, want);          // want is a multiple of 16
                    done += want;
                }
            }
        });
        pool->wait();
        if (!ok.load()) { readFailed = true; break; }
        CU(D(cuMemcpyHtoDAsync)(ctx->fileWindow, dst, (size_t)bytes, ctx->streamMain));
        uint64_t winBegin = first, winEnd = first + count;
        uint64_t chunk0 = chunkOfSample(rec, lp.plan, n, winBegin), chunk1 = chunkOfSample(rec, lp.plan, n, winEnd - 1) + 1;
        CUdeviceptr window = ctx->fileWindow;
        CU(D(cuEventRecord)(q.ev[w & 1][0], ctx->streamMain));
        rc = launch(ctx, ctx->fn[K_IMPORT_SCATTER], blocks * 2, 256, ctx->streamMain, a, window, winBegin, winEnd, chunk0, chunk1);
        if (rc) return rc;
        CU(D(cuEventRecord)(q.ev[w & 1][1], ctx->streamMain));
    }
    if (!readFailed) {
        // the voxels against the grids the points rebuilt: membership, then the two flip passes, then the counts
        CU(D(cuEventRecord)(q.ev[2][0], ctx->streamMain));
        for (uint32_t mode = 0; mode < 3; mode++) {
            rc = launch(ctx, ctx->fn[K_IMPORT_VOXELS], blocks * 2, 256, ctx->streamMain, a, numChunks, mode); if (rc) return rc;
        }
        rc = launch(ctx, ctx->fn[K_IMPORT_COUNT_GRIDS], blocks * 2, 256, ctx->streamMain, a); if (rc) return rc;
        CU(D(cuEventRecord)(q.ev[2][1], ctx->streamMain));
    }
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    for (uint64_t w = numWindows >= 2 ? numWindows - 2 : 0; w < numWindows && !readFailed; w++) { rc = retire(w); if (rc) return rc; }
    CU(D(cuEventElapsedTime)(&t, ctx->evStart, ctx->evEnd));
    ms += t;
    if (!readFailed) { CU(D(cuEventElapsedTime)(&t, q.ev[2][0], q.ev[2][1])); ms += t; }
    uint32_t error = 0;
    CU(D(cuMemcpyDtoH)(&error, errorDev, 4));
    if (readFailed || error) {
        rc = simlod_reset(ctx); if (rc) return rc;                   // an empty octree in the file's box
        if (readFailed) return fail(SIMLOD_ERR_INVALID, "read error in %s; the context holds an empty octree", path);
        return fail(SIMLOD_ERR_INVALID, "%s: samples do not fit their nodes (error %u: %u a point outside its leaf, %u a voxel off the centre of its points' cells, %u two voxels in one cell, %u a node with other than one voxel per cell its points occupy); the context holds an empty octree",
                    path, error, (uint32_t)IMPORT_ERR_POINT, (uint32_t)IMPORT_ERR_VOXEL, (uint32_t)IMPORT_ERR_DUPLICATE, (uint32_t)IMPORT_ERR_COUNT);
    }
    // Stats, and the ring: the next batch is batch batchletIndex, in slot batchletIndex % 50
    SimlodStats st = lp.stats;
    st.frameID = (uint32_t)ctx->frameCounter;
    st.allocatedBytes_momentary = scratch::TOTAL;                    // as every kernel_construct launch reports it
    CU(D(cuMemcpyHtoD)(ctx->buf.stats, &st, sizeof(st)));
    *ctx->hStats = st;
    CU(D(cuMemsetD32Async)(ctx->numBatchesUploaded, h.batchlet_index, 1, ctx->streamMain));
    CU(D(cuMemsetD8Async)(ctx->batchSizes, 0, 4 * RING_SLOTS, ctx->streamMain));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    ctx->uploaded = ctx->processed = h.batchlet_index;
    ctx->unpublished = 0;
    memset(ctx->hostSizes, 0, sizeof(ctx->hostSizes));
    if (info) *info = h.info;
    if (kernel_ms) *kernel_ms = ms;
    return SIMLOD_OK;
}

// ---- LAS writer (DESIGN.md §9.13); the encode is las_write.cu's, the octree source's gather export.cu's --------------
constexpr uint64_t LAS_HEADER_BYTES = 227;                                  // LAS 1.2 public header, no VLRs
constexpr uint64_t LAS_WINDOW_BYTES = LAS_WRITE_WINDOW * LAS_WRITE_RECORD;  // 208 MiB of records
constexpr uint64_t LAS_PIECE_BYTES = 8ull << 20;                            // a writer thread's unit of work
static_assert(LAS_WINDOW_BYTES <= POOL_BYTES / 2, "a window of records fits one half of the page-locked pool");
static_assert(LAS_WRITE_WINDOW * sizeof(SimlodPoint) <= FILE_WINDOW_BYTES, "a window of samples fits the octree file's window");
static_assert(2 * sizeof(LasWriteCtl) <= CTL_HOST_BYTES, "two control snapshots fit the pinned control word");

int ensureLasWindow(SimlodContext* ctx) {
    if (!ctx->lasWindow) {
        for (auto& half : ctx->evLas) for (CUevent& e : half) if (!e) CU(D(cuEventCreate)(&e, CU_EVENT_DEFAULT));
        CU(D(cuMemAlloc)(&ctx->lasWindow, LAS_WINDOW_BYTES + sizeof(LasWriteCtl)));
    }
    if (!ctx->hExportCtl) CU(D(cuMemHostAlloc)(&ctx->hExportCtl, CTL_HOST_BYTES, 0));
    return ensurePinnedPool(ctx);
}

bool pwriteAll(int fd, const char* src, uint64_t bytes, uint64_t at) {
    while (bytes) {
        const ssize_t r = pwrite(fd, src, bytes, (off_t)at);
        if (r <= 0) return false;
        src += r; at += (uint64_t)r; bytes -= (uint64_t)r;
    }
    return true;
}

void lasHeader(uint8_t* h, uint64_t n, const SimlodLasWriteParams& p, const double mn[3], const double mx[3]) {
    memset(h, 0, LAS_HEADER_BYTES);
    auto u16 = [&](int o, uint16_t v) { memcpy(h + o, &v, 2); };
    auto u32 = [&](int o, uint32_t v) { memcpy(h + o, &v, 4); };
    auto f64 = [&](int o, double v) { memcpy(h + o, &v, 8); };
    memcpy(h, "LASF", 4);
    h[24] = 1; h[25] = 2;                                   // version 1.2; system identifier zero bytes
    memcpy(h + 58, "simlod_b200", 11);                      // generating software, NUL-padded; creation day and year 0
    u16(94, (uint16_t)LAS_HEADER_BYTES);
    u32(96, (uint32_t)LAS_HEADER_BYTES);                    // offset to point data; 0 VLRs
    h[104] = 2;
    u16(105, (uint16_t)LAS_WRITE_RECORD);
    u32(107, (uint32_t)n);
    u32(111, (uint32_t)n);                                  // points by return [n, 0, 0, 0, 0]
    for (int a = 0; a < 3; a++) {
        f64(131 + 8 * a, p.scale[a]);
        f64(155 + 8 * a, p.offset[a]);
        f64(179 + 16 * a, mx[a]);
        f64(187 + 16 * a, mn[a]);
    }
}

int writeLas(SimlodContext* ctx, const char* path, const SimlodLasWriteParams* params, uint64_t samples, uint64_t numSamples,
             int32_t depth, SimlodLasWriteInfo* info, float* kernel_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!path || !params || !info) return fail(SIMLOD_ERR_INVALID, "null path, params or info");
    for (int a = 0; a < 3; a++) {
        if (!std::isfinite(params->scale[a]) || !(params->scale[a] > 0.0)) return fail(SIMLOD_ERR_INVALID, "LAS scale[%d] = %g must be finite and > 0", a, params->scale[a]);
        if (!std::isfinite(params->offset[a]) || !std::isfinite(params->translation[a])) return fail(SIMLOD_ERR_INVALID, "LAS offset and translation must be finite (axis %d)", a);
    }
    rc = checkAligned("LAS", {{"samples", samples, 16}}); if (rc) return rc;
    if (samples && depth >= 0) return fail(SIMLOD_ERR_INVALID, "a depth selects a cut of the octree's samples; it does not apply to a caller's array");
    rc = checkDepth("LAS", depth); if (rc) return rc;
    if (samples && numSamples > UINT32_MAX) return fail(SIMLOD_ERR_INVALID, "%llu samples: a LAS 1.2 file holds at most 2^32 - 1 points", (unsigned long long)numSamples);
    if (params->writer_threads < 1 || params->writer_threads > 64) return fail(SIMLOD_ERR_INVALID, "writer_threads %u is outside 1..64", params->writer_threads);
    // written under a temporary name and renamed once complete: a failed call leaves no file and replaces no existing one
    const std::string tmpPath = std::string(path) + ".tmp";
    int fd = open(tmpPath.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return fail(SIMLOD_ERR_INVALID, "cannot write %s", path);
    struct Closer {
        int& fd; const std::string& tmp; bool done = false;
        ~Closer() { if (fd >= 0) close(fd); if (!done) unlink(tmp.c_str()); }
    } closer{fd, tmpPath};
    memset(info, 0, sizeof(*info));
    info->first_invalid = UINT64_MAX;

    // the octree source: the export's plan and chunk-list walk, once
    const bool octree = samples == 0;
    ExportPlanned p;
    uint64_t n = numSamples;
    if (octree) {
        rc = exportPlan(ctx, depth < 0 ? (int32_t)SIMLOD_MAX_DEPTH : depth, nullptr, &p);
        info->plan_ms = p.ms;
        if (rc) return fail(rc, "%s: not written: %s", path, g_error.c_str());
        n = p.c.numSamples;
        if (n > UINT32_MAX) return fail(SIMLOD_ERR_INVALID, "%s: not written: %llu samples, a LAS 1.2 file holds at most 2^32 - 1 points", path, (unsigned long long)n);
        rc = ensureFileWindow(ctx); if (rc) return rc;
    }
    rc = ensureLasWindow(ctx); if (rc) return rc;
    const uint64_t fileSize = LAS_HEADER_BYTES + n * LAS_WRITE_RECORD;
    if (ftruncate(fd, (off_t)fileSize) != 0) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);

    // window w: gathered (octree source) and encoded on the device, copied into pool half w & 1 with its control
    // snapshot; its pieces are handed to the writers once the copy has completed and shows no invalid sample
    const uint64_t numWindows = (n + LAS_WRITE_WINDOW - 1) / LAS_WRITE_WINDOW;
    auto windowCount = [&](uint64_t w) { return std::min<uint64_t>(LAS_WRITE_WINDOW, n - w * LAS_WRITE_WINDOW); };
    auto half = [&](uint64_t w) { return (char*)ctx->pinnedPool + (w & 1) * (POOL_BYTES / 2); };
    std::vector<uint64_t> firstPiece(numWindows + 1, 0);          // pieces of windows [0, w)
    for (uint64_t w = 0; w < numWindows; w++)
        firstPiece[w + 1] = firstPiece[w] + (windowCount(w) * LAS_WRITE_RECORD + LAS_PIECE_BYTES - 1) / LAS_PIECE_BYTES;
    const uint64_t totalPieces = firstPiece[numWindows];
    std::vector<std::atomic<uint64_t>> written(numWindows);       // pieces of window w in the file
    for (auto& c : written) c.store(0);
    std::atomic<uint64_t> published{0}, nextPiece{0};             // pieces [0, published) may be written
    std::atomic<bool> abort{false}, ioError{false};
    if (!ctx->loaderPool) ctx->loaderPool = new LoaderPool();
    LoaderPool* pool = ctx->loaderPool;
    const auto tBegin = std::chrono::steady_clock::now();
    pool->run((int)params->writer_threads, [&](int) {
        for (;;) {
            const uint64_t item = nextPiece.fetch_add(1);
            if (item >= totalPieces) break;
            while (published.load() <= item && !abort.load()) std::this_thread::yield();
            if (abort.load()) break;
            const uint64_t w = (uint64_t)(std::upper_bound(firstPiece.begin(), firstPiece.end(), item) - firstPiece.begin()) - 1;
            const uint64_t bytes = windowCount(w) * LAS_WRITE_RECORD, p0 = (item - firstPiece[w]) * LAS_PIECE_BYTES;
            const uint64_t at = LAS_HEADER_BYTES + w * LAS_WINDOW_BYTES + p0;
            if (!pwriteAll(fd, half(w) + p0, std::min<uint64_t>(LAS_PIECE_BYTES, bytes - p0), at)) { ioError.store(true); abort.store(true); break; }
            written[w].fetch_add(1);
        }
    });
    // stops and joins the writers on every exit
    struct Writers {
        LoaderPool* pool; std::atomic<bool>& abort; bool joined = false;
        void join(bool stop) { if (joined) return; if (stop) abort.store(true); pool->wait(); joined = true; }
        ~Writers() { join(true); }
    } writers{pool, abort};
    const LasWriteCtl* hctl = (const LasWriteCtl*)ctx->hExportCtl;
    const CUdeviceptr records = ctx->lasWindow, ctl = ctx->lasWindow + LAS_WINDOW_BYTES;
    CU(D(cuMemsetD8Async)(ctl, 0xff, sizeof(LasWriteCtl), ctx->streamMain));
    float encodeMs = 0.0f, copyMs = 0.0f;
    auto drain = [&](uint64_t w) -> int {             // window w has been copied out: time it, check it, publish it
        CUevent* ev = ctx->evLas[w & 1];
        CU(D(cuEventSynchronize)(ev[3]));
        float e = 0.0f, c = 0.0f;
        CU(D(cuEventElapsedTime)(&e, ev[0], ev[1]));
        CU(D(cuEventElapsedTime)(&c, ev[2], ev[3]));
        encodeMs += e; copyMs += c;
        if (hctl[w & 1].firstInvalid != UINT64_MAX) {
            info->first_invalid = hctl[w & 1].firstInvalid;
            return fail(SIMLOD_ERR_INVALID, "%s: not written: sample %llu is invalid (a non-finite coordinate, or a quantised coordinate outside int32)",
                        path, (unsigned long long)info->first_invalid);
        }
        published.store(firstPiece[w + 1]);
        return SIMLOD_OK;
    };
    const unsigned maxBlocks = (unsigned)ctx->numSMs * 8;
    for (uint64_t w = 0; w < numWindows; w++) {
        const uint64_t a = w * LAS_WRITE_WINDOW, count = windowCount(w);
        CUevent* ev = ctx->evLas[w & 1];
        CU(D(cuEventRecord)(ev[0], ctx->streamMain));
        CUdeviceptr src = (CUdeviceptr)samples + a * sizeof(SimlodPoint);
        if (octree) {
            CUdeviceptr window = ctx->fileWindow;
            uint64_t b = a + count;
            rc = launch(ctx, ctx->fn[K_EXPORT_GATHER_WINDOW], (unsigned)ctx->numSMs * 4, 256, ctx->streamMain, p.s.items, window, p.s.ctl, a, b);
            if (rc) return rc;
            src = window;
        }
        LasEncodeArgs args{devPtr(src), devPtr(records), devPtr(ctl), a, count, {}, {}, {}};
        for (int k = 0; k < 3; k++) { args.scale[k] = params->scale[k]; args.offset[k] = params->offset[k]; args.translation[k] = params->translation[k]; }
        const unsigned grid = (unsigned)std::min<uint64_t>(maxBlocks, (count + LAS_WRITE_TILE - 1) / LAS_WRITE_TILE);
        rc = launch(ctx, ctx->fn[K_LAS_ENCODE], grid, LAS_WRITE_TILE, ctx->streamMain, args); if (rc) return rc;
        CU(D(cuEventRecord)(ev[1], ctx->streamMain));
        // pool half w & 1 is free once every piece of window w - 2 is in the file
        if (w >= 2) {
            while (written[w - 2].load() < firstPiece[w - 1] - firstPiece[w - 2] && !abort.load()) std::this_thread::yield();
            if (ioError.load()) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);
        }
        CU(D(cuEventRecord)(ev[2], ctx->streamMain));
        CU(D(cuMemcpyDtoHAsync)(half(w), records, (size_t)(count * LAS_WRITE_RECORD), ctx->streamMain));
        CU(D(cuMemcpyDtoHAsync)((void*)(hctl + (w & 1)), ctl, sizeof(LasWriteCtl), ctx->streamMain));
        CU(D(cuEventRecord)(ev[3], ctx->streamMain));
        if (w > 0) { rc = drain(w - 1); if (rc) return rc; }
    }
    if (numWindows > 0) { rc = drain(numWindows - 1); if (rc) return rc; }
    writers.join(false);
    if (ioError.load()) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);

    // the header last, once the bounds are known: double(q) * scale + offset, multiply then add
    double mn[3] = {0.0, 0.0, 0.0}, mx[3] = {0.0, 0.0, 0.0};
    if (n > 0) {
        const LasWriteCtl& c = hctl[(numWindows - 1) & 1];
        for (int a = 0; a < 3; a++) {
            const int32_t qmin = (int32_t)(c.qmin[a] ^ 0x80000000u), qmax = (int32_t)(~c.qmaxInv[a] ^ 0x80000000u);
            volatile double lo = (double)qmin * params->scale[a], hi = (double)qmax * params->scale[a];   // no contraction
            mn[a] = lo + params->offset[a];
            mx[a] = hi + params->offset[a];
        }
    }
    uint8_t head[LAS_HEADER_BYTES];
    lasHeader(head, n, *params, mn, mx);
    if (!pwriteAll(fd, (const char*)head, LAS_HEADER_BYTES, 0)) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);
    const int closed = close(fd);
    fd = -1;
    if (closed != 0) return fail(SIMLOD_ERR_INVALID, "write error in %s", path);
    if (rename(tmpPath.c_str(), path) != 0) return fail(SIMLOD_ERR_INVALID, "cannot write %s (rename from %s failed)", path, tmpPath.c_str());
    closer.done = true;
    info->num_points = n;
    info->file_size = fileSize;
    for (int a = 0; a < 3; a++) { info->min[a] = mn[a]; info->max[a] = mx[a]; }
    info->encode_ms = encodeMs;
    info->copy_ms = copyMs;
    info->write_ms = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tBegin).count();
    info->num_windows = (uint32_t)numWindows;
    if (kernel_ms) *kernel_ms = info->plan_ms + encodeMs;
    return SIMLOD_OK;
}
}  // namespace

extern "C" {

int simlod_write_las(SimlodContext* ctx, const char* path, const SimlodLasWriteParams* params, uint64_t samples,
                     uint64_t num_samples, int32_t depth, SimlodLasWriteInfo* info, float* kernel_ms) {
    return writeLas(ctx, path, params, samples, num_samples, depth, info, kernel_ms);
}

int simlod_read_octree_header(const char* path, SimlodOctreeFileHeader* out) {
    if (!path || !out) return fail(SIMLOD_ERR_INVALID, "null argument");
    return readOctreeHeader(path, out);
}

int simlod_save_octree(SimlodContext* ctx, const char* path, SimlodExportInfo* info, float* kernel_ms) {
    return saveOctree(ctx, path, info, kernel_ms);
}

int simlod_load_octree(SimlodContext* ctx, const char* path, int loader_threads, SimlodExportInfo* info, float* kernel_ms) {
    return loadOctree(ctx, path, loader_threads, info, kernel_ms);
}

// ---- spatial exchange (SURVEY.md §8f-3); kernels in partition.cu ----------------------------------------
namespace {
constexpr uint32_t PART_SLOTS = 64;
using part::MAX_RANKS;
using part::MAX_CELLS;

// per counted batch: blockHist[blocks][8] | blockBase[blocks][8] | totals[8] | cellCounts[512]
uint64_t partSlotBytes(uint32_t blocks) { return (uint64_t)blocks * MAX_RANKS * 4 * 2 + MAX_RANKS * 4 + MAX_CELLS * 4; }
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
    if (plan->num_ranks < 1 || plan->num_ranks > MAX_RANKS) return fail(SIMLOD_ERR_INVALID, "partition over %u ranks (1..8)", plan->num_ranks);
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
    p->perBlock = std::max(part::BLOCK, (per + part::BLOCK - 1) / part::BLOCK * part::BLOCK);
    memset(p->owner, 0, sizeof(p->owner));
    memcpy(p->owner, plan->owner, numCells);
    return partScratchEnsure(ctx);
}

// the slot simlod_partition_count counted this batch into, PART_SLOTS if none
uint32_t partSlotOf(const SimlodContext* ctx, uint64_t points, uint32_t count) {
    uint32_t slot = PART_SLOTS;
    for (uint32_t i = 0; i < PART_SLOTS; i++)
        if (ctx->partSlots[i].valid && ctx->partSlots[i].points == points && ctx->partSlots[i].count == count) slot = i;
    return slot;
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
    uint32_t slot = partSlotOf(ctx, device_points, count);
    if (slot == PART_SLOTS) { slot = ctx->partNextSlot; ctx->partNextSlot = (ctx->partNextSlot + 1) % PART_SLOTS; }
    CUdeviceptr pts = (CUdeviceptr)device_points;
    CUdeviceptr blockHist = ctx->partScratch + partSlotBytes(blocks) * slot, blockBase = blockHist + (size_t)blocks * MAX_RANKS * 4,
                totals = blockBase + (size_t)blocks * MAX_RANKS * 4, cells = totals + MAX_RANKS * 4;
    CU(D(cuMemsetD8Async)(cells, 0, MAX_CELLS * 4, ctx->streamMain));
    rc = launch(ctx, ctx->fn[K_PART_COUNT], blocks, part::BLOCK, ctx->streamMain, p, pts, blockHist, cells); if (rc) return rc;
    rc = launch(ctx, ctx->fn[K_PART_SCAN], 1, part::BLOCK, ctx->streamMain, blockHist, blocks, blockBase, totals); if (rc) return rc;
    uint32_t host[MAX_RANKS + MAX_CELLS];
    CU(D(cuMemcpyDtoHAsync)(host, totals, sizeof(host), ctx->streamMain));
    CU(D(cuStreamSynchronize)(ctx->streamMain));
    for (uint32_t d = 0; d < plan->num_ranks; d++) rank_counts[d] = host[d];
    if (cell_counts) for (uint32_t c = 0; c < (1u << (3 * plan->level)); c++) cell_counts[c] = host[MAX_RANKS + c];
    ctx->partSlots[slot].points = device_points; ctx->partSlots[slot].count = count; ctx->partSlots[slot].valid = true;
    return SIMLOD_OK;
}

int simlod_partition_scatter(SimlodContext* ctx, uint64_t device_points, uint32_t count, const SimlodPartitionPlan* plan,
                             const uint64_t* dest_ptrs, const uint64_t* dest_offsets, const uint64_t* signal_ptrs, uint32_t signal_value) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!dest_ptrs || !dest_offsets) return fail(SIMLOD_ERR_INVALID, "null argument");
    const uint32_t slot = partSlotOf(ctx, device_points, count);
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
    CUdeviceptr blockBase = ctx->partScratch + partSlotBytes(blocks) * slot + (size_t)blocks * MAX_RANKS * 4;
    CUdeviceptr blocksDone = ctx->partScratch + partSlotBytes(blocks) * PART_SLOTS;
    rc = launch(ctx, ctx->fn[K_PART_SCATTER], blocks, part::BLOCK, ctx->streamMain, p, t, pts, blockBase, blocksDone); if (rc) return rc;
    ctx->partSlots[slot].valid = false;
    return SIMLOD_OK;
}

int simlod_partition_wait(SimlodContext* ctx, uint64_t local_flags, uint32_t num_ranks, uint32_t value, uint32_t timeout_ms) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!local_flags || num_ranks < 1 || num_ranks > MAX_RANKS) return fail(SIMLOD_ERR_INVALID, "bad flags / rank count");
    { int rcs = partScratchEnsure(ctx); if (rcs) return rcs; }
    CUdeviceptr flags = (CUdeviceptr)local_flags;
    CUdeviceptr timedOut = ctx->partScratch + partSlotBytes((uint32_t)ctx->numSMs * 4) * PART_SLOTS + 4;
    uint64_t cycles = (uint64_t)(timeout_ms ? timeout_ms : 10000) * 2000000ull;          // SM clock ~2 GHz
    rc = launch(ctx, ctx->fn[K_PART_WAIT], 1, 32, ctx->streamMain, flags, num_ranks, value, cycles, timedOut); if (rc) return rc;
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

int simlod_export_framebuffer(SimlodContext* ctx, uint64_t dst_device) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!dst_device) return fail(SIMLOD_ERR_INVALID, "null destination");
    CU(D(cuMemcpyDtoDAsync)((CUdeviceptr)dst_device, ctx->buf.renderbuffer + rbuf::OFF_FB, (size_t)ctx->cfg.width * ctx->cfg.height * 8, ctx->streamMain));
    return SIMLOD_OK;
}

int simlod_peer_signal(SimlodContext* ctx, const uint64_t* signal_ptrs, uint32_t num_ranks, uint32_t value) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!signal_ptrs || num_ranks < 1 || num_ranks > MAX_RANKS) return fail(SIMLOD_ERR_INVALID, "bad signal words / rank count");
    SignalArgs a;
    memset(&a, 0, sizeof(a));
    for (uint32_t d = 0; d < num_ranks; d++) { if (!signal_ptrs[d]) return fail(SIMLOD_ERR_INVALID, "null signal word for rank %u", d); a.signal[d] = signal_ptrs[d]; }
    a.numRanks = num_ranks; a.value = value;
    return launch(ctx, ctx->fn[K_PEER_SIGNAL], 1, 32, ctx->streamMain, a);
}

int simlod_composite_framebuffers(SimlodContext* ctx, const uint64_t* fb_ptrs, uint32_t num_ranks, uint32_t rank,
                                  const uint64_t* signal_ptrs, uint32_t signal_value) {
    int rc = setCurrent(ctx); if (rc) return rc;
    if (!fb_ptrs || num_ranks < 1 || num_ranks > MAX_RANKS || rank >= num_ranks) return fail(SIMLOD_ERR_INVALID, "bad framebuffer list / rank");
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
    return launch(ctx, ctx->fn[K_COMPOSITE], (unsigned)ctx->numSMs * 4, part::BLOCK, ctx->streamMain, a, blocksDone);
}

}  // extern "C"
