// simlod_b200.h — C ABI of the H100-native SimLOD hot path.
//
// The reference has no C library boundary: its host (modules/progressive_octree/
// main_progressive_octree.cpp) compiles three CUDA programs at run time through
// CudaModularProgram (include/CudaModularProgram.h:140-264) and launches the kernels they export
// with cuLaunchCooperativeKernel. This header is that launch surface restated headless (no
// OpenGL window, no loader threads): each entry point names the reference function it replaces.
// Plain pointers and sizes only; no C++ or torch types cross the boundary.
//
// The kernels themselves (kernel_construct, kernel_render, kernel) keep the reference's names and
// argument lists, so a cubin built from simlod_b200/csrc can equally be loaded by the reference's
// own host through its kernels[name] map (see INTEGRATION.md).
#pragma once
#include <stdint.h>
#include "simlod_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct SimlodContext SimlodContext;

enum {
    SIMLOD_OK                = 0,
    SIMLOD_ERR_CUDA          = -1,   // a CUDA driver call failed; see simlod_last_error()
    SIMLOD_ERR_INVALID       = -2,   // bad argument
    SIMLOD_ERR_RING_FULL     = -3,   // all 50 ring slots hold unprocessed batches (back-pressure, main.cpp:820,1012)
    SIMLOD_ERR_MODULE        = -4,   // cubin could not be loaded or lacks the required kernel
    SIMLOD_ERR_CAPACITY      = -5,   // persistent heap almost full: the device stopped consuming batches (Stats::memCapacityReached)
    SIMLOD_ERR_OVERFLOW      = -6,   // kernel_construct exceeded one of its per-batch capacities (Stats::dbg, sticky until the next reset)
};

enum {  // Stats::dbg after kernel_construct (the reference leaves the field at 0): sticky until the next reset
    SIMLOD_DBG_SPLIT_POSTPONED_SPILL = 1 << 0,   // > 3 Mi spilled points in one batch: a split waits for the next batch (octree exact, a leaf holds > 50 000 points for now)
    SIMLOD_DBG_VOXELS_DROPPED        = 1 << 1,   // > 4 Mi voxels created in one batch
    SIMLOD_DBG_DIRECTORY_FULL        = 1 << 2,   // chunk directory of one batch exhausted: voxels dropped
    SIMLOD_DBG_SPLIT_POSTPONED_NODES = 1 << 3,   // nodes[] (40 MB = 263 157 nodes) full: a split was refused
    SIMLOD_DBG_CHUNK_STACK_FULL      = 1 << 4,   // free-chunk stack full: freed chunks leaked
    SIMLOD_DBG_SPLIT_POSTPONED_COUNT = 1 << 5,   // > 100 000 splits in one batch
    SIMLOD_DBG_ROWS_FULL             = 1 << 6,   // > 65 536 non-empty leaves at once (or a leaf beyond 64 chunks): points dropped
    SIMLOD_DBG_FAR_POINT             = 1 << 7,   // informational: a point > 16 cube edges outside the box took the exhaustive sampling path
    SIMLOD_DBG_INTERNAL              = 1 << 8,   // an invariant of the builder failed
    SIMLOD_DBG_FATAL_MASK            = 0x156,    // the bits for which simlod_update_octree / simlod_insert* return SIMLOD_ERR_OVERFLOW
};

enum {  // the three CUDA programs of main_progressive_octree.cpp:603-626
    SIMLOD_PROGRAM_CONSTRUCT = 0,    // exports kernel_construct
    SIMLOD_PROGRAM_RENDER    = 1,    // exports kernel_render
    SIMLOD_PROGRAM_RESET     = 2,    // exports kernel
};

typedef struct SimlodConfig {
    int32_t  device;                  // CUDA ordinal (reference: always 0, main.cpp:274)
    uint32_t width, height;           // render target; replaces the GL colour attachment (main.cpp:472-486)
    uint64_t momentary_bytes;         // 0 -> 300 000 000 (main.cpp:554). The reference kernels need >= 408 800 192.
    uint64_t nodes_bytes;             // 0 ->  40 000 000 (main.cpp:552-555)
    uint64_t renderbuffer_bytes;      // 0 -> 200 000 000 (main.cpp:556)
    uint64_t persistent_bytes;        // 0 -> 80 % of free device memory (main.cpp:584)
    int32_t  construct_blocks_per_sm; // 0 -> occupancy query; 1 = the reference's launch shape (main.cpp:370-371)
    int32_t  render_blocks_per_sm;    // 0 -> occupancy query (main.cpp:493-497)
} SimlodConfig;

// initCuda + initCudaProgram (main.cpp:272-281, 549-642): context, streams, events, all device
// buffers, the three programs (built-in sm_90a cubins), and a surface-capable RGBA8 array.
int  simlod_create(const SimlodConfig* config, SimlodContext** out);
void simlod_destroy(SimlodContext* ctx);
const char* simlod_last_error(void);

// CudaModularProgram's module map / hot reload (CudaModularProgram.h:166-190,245-252): replace one
// program by a cubin file that exports the same kernel name; NULL restores the built-in program.
// This is how the tests run the reference's own kernels on the same buffers.
int simlod_use_module(SimlodContext* ctx, int program, const char* cubin_path);

// getUniforms (main.cpp:283-331). The caller fills camera matrices, box and settings; the
// library overwrites width/height and the two buffer capacities with its own values.
int simlod_set_uniforms(SimlodContext* ctx, const SimlodUniforms* uniforms);
int simlod_get_uniforms(SimlodContext* ctx, SimlodUniforms* out);

// resetCUDA (main.cpp:333-361). Also clears nodes[] first (the reference relies on a zeroed allocation).
int simlod_reset(SimlodContext* ctx);
// same with an explicit launch shape of the reset kernel; (1, 1) is the reference's own (main.cpp:348-354),
// simlod_reset uses one 256-thread block per SM (the kernel is grid-stride)
int simlod_reset_with_grid(SimlodContext* ctx, uint32_t blocks, uint32_t threads);

// spawnUploader's inner step (main.cpp:1033-1056): copy one batch (<= 1 000 000 points) into ring
// slot (uploaded % 50) on the upload stream, then publish batchSizes[slot] and numBatchesUploaded.
// Asynchronous when `points` is page-locked. SIMLOD_ERR_RING_FULL if 50 batches are pending.
int simlod_upload_batch(SimlodContext* ctx, const SimlodPoint* host_points, uint32_t count);
// same, source already in device memory (device-to-device copy)
int simlod_upload_batch_device(SimlodContext* ctx, uint64_t device_points, uint32_t count);

// updateOctree (main.cpp:364-428): ONE cooperative launch of kernel_construct, timed with an event
// pair as the reference does (main.cpp:394,408-421). Consumes up to 20 uploaded batches or 10 ms.
// Blocks until the launch has finished; *kernel_ms (optional) receives the event time.
int simlod_update_octree(SimlodContext* ctx, float* kernel_ms);

// The main loop's streaming behaviour (main.cpp:1176-1180 + uploader thread) for a point set in
// host memory: uploads in 1 000 000-point batches overlapped with update launches until every
// point is inserted. *kernel_ms (optional) = sum of kernel_construct event times (the reference's
// "points/sec update kernel" denominator, main.cpp:1484); *total_ms (optional) = device time from
// the first upload to the end of the last launch, measured with an event pair on the launch stream.
int simlod_insert(SimlodContext* ctx, const SimlodPoint* host_points, uint64_t count, float* kernel_ms, float* total_ms);
// same with the whole point set resident in device memory: the kernel reads the 1 000 000-point batches where they are
// (no copy into the ring; the `points` argument of each launch maps the ring slots of its 50-batch window onto the
// caller's buffer, which must stay valid and unchanged until the call returns)
int simlod_insert_device(SimlodContext* ctx, uint64_t device_points, uint64_t count, float* kernel_ms, float* total_ms);

// Streaming front end for one `.simlod` file (SURVEY.md §8f-1): reload() + spawnLoader + spawnUploader of
// main.cpp:644-760, 811-958, 963-1063. The 24-byte header (6 x f32 min, max; tools/las2simlod.mjs:95-101)
// gives the box (boxMin = 0, boxMax = max - min, main.cpp:312-313); the octree is reset; `loader_threads`
// host threads read 1 000 000-point batches (loadFileNative, SimlodLoader.cpp:147-157) into a pool of pinned
// slots (main.cpp:141-222) while the uploader publishes them IN FILE ORDER and update launches consume them.
int simlod_insert_simlod_file(SimlodContext* ctx, const char* path, int loader_threads, uint64_t* num_points,
                              float* kernel_ms, float* total_ms);
// same with flags. SIMLOD_STREAM_DIRECT: unbuffered (O_DIRECT) reads of whole 4 KB blocks — the reference's Windows
// loader reads unbuffered too (SimlodLoader.cpp:59-141, FILE_FLAG_NO_BUFFERING) — for files that are not in the page
// cache; SIMLOD_ERR_INVALID when the file system cannot do it (tmpfs).
enum { SIMLOD_STREAM_DIRECT = 1 };
int simlod_insert_simlod_file_ex(SimlodContext* ctx, const char* path, int loader_threads, uint32_t flags, uint64_t* num_points,
                                 float* kernel_ms, float* total_ms);

// LAS front end (SURVEY.md §8f-2). The reference decodes LAS point records on CPU threads
// (loadLasNative, LasLoader.cpp:169-226) and uploads 16-byte points; here the raw records are uploaded
// and decoded on the device straight into the next ring slot, then published like any batch.
// `format` selects the RGB offset as the reference does (2 -> 20, 3/5 -> 28, 7 -> 30, else no colour);
// x = double(X) * scale + (offset + translation), narrowed to float (LasLoader.cpp:199-210).
typedef struct SimlodLasLayout {
    uint32_t bytes_per_point;       // LasHeader::bytesPerPoint (<= 96)
    uint32_t format;                // LasHeader::format
    double   scale[3];
    double   offset[3];
    double   translation[3];        // the host passes -min (main.cpp:868-873), so that boxMin = 0
} SimlodLasLayout;
int simlod_upload_batch_las(SimlodContext* ctx, const void* host_records, uint32_t count, const SimlodLasLayout* layout);
int simlod_upload_batch_las_device(SimlodContext* ctx, uint64_t device_records, uint32_t count, const SimlodLasLayout* layout);

// renderCUDA (main.cpp:465-546): one cooperative launch of kernel_render into the surface.
int simlod_render(SimlodContext* ctx, float* kernel_ms);

// Stats read-back (main.cpp:1201-1216)
int simlod_get_stats(SimlodContext* ctx, SimlodStats* out);
// packed depth|colour framebuffer, width*height u64 (render buffer byte 31 200 144, render.cu:1122-1123)
int simlod_read_framebuffer(SimlodContext* ctx, uint64_t* out);
// RGBA8 surface written by kernel_render, width*height u32 (what the reference displays)
int simlod_read_surface(SimlodContext* ctx, uint32_t* out);

// Raw access for tests and tools: device addresses and sizes of the buffers the kernels share
// (nodes[], persistent heap, momentary buffer, render buffer, point ring) and a bounded copy.
typedef struct SimlodBuffers {
    uint64_t nodes, nodes_bytes;
    uint64_t persistent, persistent_bytes;
    uint64_t momentary, momentary_bytes;
    uint64_t renderbuffer, renderbuffer_bytes;
    uint64_t ring, ring_bytes;
    uint64_t stats;
} SimlodBuffers;
int simlod_get_buffers(SimlodContext* ctx, SimlodBuffers* out);
int simlod_memcpy_dtoh(SimlodContext* ctx, void* dst, uint64_t src_device, uint64_t bytes);
int simlod_memcpy_htod(SimlodContext* ctx, uint64_t dst_device, const void* src, uint64_t bytes);

// pinned host memory (the reference's pinned pool, main.cpp:141-222) and plain device memory
int simlod_host_alloc(SimlodContext* ctx, uint64_t bytes, void** out);
int simlod_host_free(SimlodContext* ctx, void* ptr);
int simlod_device_alloc(SimlodContext* ctx, uint64_t bytes, uint64_t* out);
int simlod_device_free(SimlodContext* ctx, uint64_t ptr);

// host NUMA node the context's page-locked buffers (simlod_host_alloc, the streamer's pool) were placed on: the node
// closest to the device (CU_DEVICE_ATTRIBUTE_HOST_NUMA_ID, else sysfs); -1 when unknown or before the first allocation
int simlod_get_numa_node(SimlodContext* ctx, int* node);
// launch bookkeeping: kernels launched by this context so far, and the grid sizes in use
int simlod_get_launch_info(SimlodContext* ctx, uint64_t* launches, uint32_t* construct_blocks, uint32_t* render_blocks, uint32_t* num_sms);
// MUFU.RCP(x) as the device computes it (the one float a CPU restatement cannot derive when the
// octree cube size is not a power of two; see oracle/)
int simlod_device_rcp(SimlodContext* ctx, float x, float* out);
// Synthetic point streams of the benchmark configurations generated on the device (bench / test
// infrastructure; restates simlod_b200/data.py, see csrc/gen.cu): points [first, first + count) of an
// n_total-point stream into device_points. `size` is the cube edge of SIMLOD_GEN_UNIFORM (ignored otherwise).
enum { SIMLOD_GEN_UNIFORM = 0, SIMLOD_GEN_TERRAIN = 1, SIMLOD_GEN_SHELL = 2 };
int simlod_generate(SimlodContext* ctx, int kind, uint64_t n_total, uint64_t first, uint64_t count, uint64_t seed, float size, uint64_t device_points);
// wait for everything this context has enqueued (uploads, decodes, launches)
int simlod_synchronize(SimlodContext* ctx);
// flush the L2 cache by overwriting a scratch buffer larger than it (bench hygiene)
int simlod_flush_l2(SimlodContext* ctx);

// ---- spatial exchange for ONE octree over several GPUs (SURVEY.md §8f-3; no counterpart in the reference,
// which builds on one GPU). Rank r owns the level-`level` cells c of the octree cube with owner[c] == r; a point's
// cell is decided with the builder's own quantisation (voxels.cu:148-155, child index per level voxels.cu:171-179;
// cell = child indices root first, 3 bits per level), against the box of simlod_set_uniforms.
typedef struct SimlodPartitionPlan {
    uint32_t level;               /* 1..3 */
    uint32_t num_ranks;           /* 1..8 */
    uint8_t owner[512];           /* [8^level] cell -> rank */
} SimlodPartitionPlan;
// pass 1: how many of the `count` points at device_points go to each rank (rank_counts[num_ranks]); cell_counts
// (optional, [8^level]) receives the per-cell histogram used to plan owners. Synchronous.
int simlod_partition_count(SimlodContext* ctx, uint64_t device_points, uint32_t count, const SimlodPartitionPlan* plan,
                           uint64_t* rank_counts, uint64_t* cell_counts);
// pass 2 (after pass 1 on the same points / count; up to 64 counted batches may be outstanding): stable scatter.
// The k-th point of the batch that belongs to rank d is stored at ((SimlodPoint*)dest_ptrs[d])[dest_offsets[d] + k];
// dest_ptrs may be local device memory or peer memory mapped over NVLink (the store stream IS the exchange).
// signal_ptrs (optional, [num_ranks]): this sender's 32-bit flag word in every destination; once all stores of
// the launch are visible system-wide the kernel releases signal_value into each of them. Asynchronous on the
// launch stream.
int simlod_partition_scatter(SimlodContext* ctx, uint64_t device_points, uint32_t count, const SimlodPartitionPlan* plan,
                             const uint64_t* dest_ptrs, const uint64_t* dest_offsets, const uint64_t* signal_ptrs, uint32_t signal_value);
// receiving side: returns when every sender's flag in local_flags[0..num_ranks) has reached `value` (wrap-around
// compare), i.e. all buckets of that step have landed here; everything enqueued on this context before the call
// has completed too. SIMLOD_ERR_CUDA naming the silent rank after timeout_ms (0 = 10 s).
int simlod_partition_wait(SimlodContext* ctx, uint64_t local_flags, uint32_t num_ranks, uint32_t value, uint32_t timeout_ms);

// ---- depth compositing of the ranks' packed framebuffers over peer memory (SURVEY.md §8e/§8f-3). The u64 word
// is depth << 32 | colour (render.cu:61-104 of the reference), so an element-wise unsigned minimum over the ranks
// is the depth test one GPU's atomicMin performs on the union of the samples.
// copy this context's packed framebuffer (width x height u64) to dst_device, e.g. a peer-visible buffer; async
int simlod_export_framebuffer(SimlodContext* ctx, uint64_t dst_device);
// release `value` into this rank's flag word in every peer, behind everything enqueued so far; async
int simlod_peer_signal(SimlodContext* ctx, const uint64_t* signal_ptrs, uint32_t num_ranks, uint32_t value);
// two-shot all-reduce(min) in one kernel: this rank reduces slice `rank` of all fb_ptrs[0..num_ranks) (peer loads)
// and stores the result into slice `rank` of all of them (peer stores), then releases signal_value into
// signal_ptrs (optional). Callers order it after every peer's simlod_peer_signal with simlod_partition_wait and
// wait for every peer's completion flag the same way. Asynchronous.
int simlod_composite_framebuffers(SimlodContext* ctx, const uint64_t* fb_ptrs, uint32_t num_ranks, uint32_t rank,
                                  const uint64_t* signal_ptrs, uint32_t signal_value);

#ifdef __cplusplus
}
#endif
