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
// Records from host memory are copied into a ring of device staging slots on a copy stream of their own; the decode
// waits for its copy, so the copies of later batches keep the PCIe link busy while an update launch occupies the SMs.
int simlod_upload_batch_las(SimlodContext* ctx, const void* host_records, uint32_t count, const SimlodLasLayout* layout);
int simlod_upload_batch_las_device(SimlodContext* ctx, uint64_t device_records, uint32_t count, const SimlodLasLayout* layout);

// The LAS public header fields the reference reads (loadHeader, LasLoader.h:21-55); layout in simlod_abi.h.
// SIMLOD_ERR_INVALID naming the file when it cannot be read, is shorter than its header or lacks the LASF signature.
// Needs no context and no GPU.
int simlod_read_las_header(const char* path, SimlodLasHeader* out);

// reload() of the reference for a list of point-cloud files (main.cpp:644-773, 811-958; onFileDrop, :1120-1150):
// `.las` and `.simlod` files, by extension, compared case-insensitively. Every path, header and file size is checked
// first; on any error the call returns SIMLOD_ERR_INVALID naming the file and leaves the octree, Stats and uniforms as
// they were (a missing file, an unknown extension, `.laz`, no LASF signature, a record size or format the decoder
// rejects, records past the end of the file, a `.simlod` file shorter than its 24-byte header). Then:
//   box        the union of float(header min / max) of the LAS files and the header floats of the .simlod files;
//              the uniforms get boxMin = 0, boxMax = max - min (float), and the octree is reset
//   batches    each file in list order is cut into ceil(n / 1 000 000) batches, the last one partial; a file without
//              points adds its box and no batch
//   decode     LAS records are decoded on the device with translation = -boxMin (simlod_upload_batch_las: alpha 0xff,
//              RGB for formats 2, 3, 5 and 7 only); .simlod points are inserted as they are stored
// `loader_threads` host threads read ~1 MB pieces of the files in list order into a 512 MB page-locked pool; batches are
// published in list order. *num_points, *kernel_ms, *total_ms and SIMLOD_STREAM_DIRECT (for every file) as for
// simlod_insert_simlod_file_ex.
int simlod_insert_files(SimlodContext* ctx, const char* const* paths, uint32_t num_paths, int loader_threads,
                        uint32_t flags, uint64_t* num_points, float* kernel_ms, float* total_ms);

// renderCUDA (main.cpp:465-546): one cooperative launch of kernel_render into the surface. With a clip set
// (simlod_set_clip) the launch is of simlod_render_clip instead, on the same grid; SIMLOD_ERR_MODULE, with nothing
// launched, when the render program is a module without that entry point.
int simlod_render(SimlodContext* ctx, float* kernel_ms);

// Stats read-back (main.cpp:1201-1216)
int simlod_get_stats(SimlodContext* ctx, SimlodStats* out);
// packed depth|colour framebuffer, width*height u64 (render buffer byte 31 200 144, render.cu:1122-1123)
int simlod_read_framebuffer(SimlodContext* ctx, uint64_t* out);
// RGBA8 surface written by kernel_render, width*height u32 (what the reference displays)
int simlod_read_surface(SimlodContext* ctx, uint32_t* out);

// Octree export: the node hierarchy and its samples as flat arrays in device memory, read from the ABI alone (Node
// children, points / numPoints, voxelChunks / numVoxelsStored; up to 1000 samples per chunk, in chunk-list order), so it
// works the same on an octree built by the reference kernels. A snapshot of the octree as the last completed
// kernel_construct left it; it writes nothing into the context's buffers or Stats.
//   depth < 0        every node, with its points and its voxels (SIMLOD_EXPORT_SAMPLED on every record)
//   0 <= depth <= 20 records for the nodes of level <= depth; samples for the cut at `depth`: the voxels of each inner
//                    node at level == depth and the points of each leaf at level <= depth (each region covered once)
// dst_nodes receives SimlodExportNode records (node_capacity of them), dst_samples 16-byte SimlodPoint samples
// (sample_capacity of them); both device addresses, 16-byte aligned. With dst_nodes == dst_samples == 0 only *info is
// filled (size query). SIMLOD_ERR_INVALID, with nothing written to dst_*, for a capacity below *info's counts, depth > 20
// or an inconsistent image (a child pointer outside nodes[], an inner node without 8 children, a chunk pointer outside
// the used heap, a list shorter than its count). Enqueued on the launch stream; returns once the export has completed.
// *kernel_ms (optional) = event time of the export kernels. Scratch memory is the context's, kept until simlod_destroy.
int simlod_export_octree(SimlodContext* ctx, int32_t depth, uint64_t dst_nodes, uint64_t node_capacity,
                         uint64_t dst_samples, uint64_t sample_capacity, SimlodExportInfo* info, float* kernel_ms);

// View export: the LOD cut simlod_render draws for the current uniforms (transform_updateBound, so a frozen visibility
// transform is honoured; width, height, minNodeSize, the box), in the records and samples of simlod_export_octree. A node
// is drawn when it is visible and either a large leaf, or not large with a large parent, evaluated per node of
// nodes[0, Stats::numNodes) by the renderer's own arithmetic. Records: the root and the 8 children of every inner node
// with a drawn node strictly below it, breadth-first; SIMLOD_EXPORT_SAMPLED exactly on the drawn nodes, which carry their
// points and their stored voxels; the others carry none. Nothing drawn: the root record alone. Render-time colouring does
// not apply. Destinations, size query, errors and scratch as for simlod_export_octree; a drawn node the breadth-first
// pass does not reach is reported as a child pointer error. Unlike simlod_render it writes nothing into nodes[] (not
// even the visible / isLarge flags) or any other buffer of the context.
int simlod_export_view(SimlodContext* ctx, uint64_t dst_nodes, uint64_t node_capacity, uint64_t dst_samples,
                       uint64_t sample_capacity, SimlodExportInfo* info, float* kernel_ms);

// Region query (DESIGN.md §9.8): the samples of the octree inside a box, a sphere or a convex set of half-spaces, filtered
// on the device into a flat array of 16-byte SimlodPoint samples. Coordinates are those of the stored samples (the ones
// the insert calls received, the box of simlod_set_uniforms).
// SimlodRegion (a box, a sphere or up to SIMLOD_REGION_MAX_PLANES half-spaces): layout in simlod_abi.h.
typedef struct SimlodQueryInfo {
    uint64_t num_samples, num_points, num_voxels;   //   0  returned
    uint64_t samples_tested;                        //  24  samples of the visited nodes, each put through the per-sample test
    uint32_t nodes_visited;                         //  32  sampled nodes the region may touch (the rest were skipped unread)
    uint32_t max_level;                             //  36  deepest level in the octree
} SimlodQueryInfo;
SIMLOD_STATIC_ASSERT(sizeof(SimlodQueryInfo) == 40, "QueryInfo");
SIMLOD_STATIC_ASSERT(offsetof(SimlodQueryInfo, samples_tested) == 24 && offsetof(SimlodQueryInfo, nodes_visited) == 32, "QueryInfo.samples_tested");
//   sample set   depth < 0: the points of every leaf, i.e. the inserted point set, no voxels. 0 <= depth <= 20: the cut of
//                simlod_export_octree at `depth` (the voxels of each inner node at level == depth, the points of each
//                leaf at level <= depth), so a coarse preview of a region costs a coarse amount of work
//   result       exactly those samples of the set that pass the region's predicate above and are eligible (below),
//                bit for bit as stored. Order: nodes in the export's breadth-first (level, Morton) order, within a node in
//                chunk-list order; two queries of the same buffers are byte-identical
//   predicates   evaluated in float32 without contraction: six comparisons for the box;
//                (x-cx)*(x-cx) + (y-cy)*(y-cy) + (z-cz)*(z-cz) <= r*r, summed left to right, for the sphere;
//                ((nx*x + ny*y) + nz*z) + d >= 0 for each plane, used as given (not normalised)
//   eligible     a point is eligible when on every axis it is not below boxMin and its lattice coordinate, the builder's
//                u32(2^20 * (p - boxMin) * rcp(cubeSize)), is below 2^20. The builder files a point outside that
//                half-open cube under a wrapped or saturated coordinate, so no node's box bounds it and no hierarchical
//                skip could be exact for it: such points (in practice those exactly on the max face of the longest axis)
//                are never returned. Voxel centres are always eligible.
// A node whose box, inflated by a rounding margin, cannot hold an eligible sample that passes is skipped with its
// subtree, unread; every sample of the other (visited) nodes is tested. dst_samples == 0 fills *info only (size query).
// SIMLOD_ERR_INVALID, before any launch, for depth > 20, a misaligned destination or a malformed region (unknown kind,
// num_planes 0 or > 16, a non-finite number, box_min > box_max on an axis, a negative radius); with nothing written,
// for a capacity below info->num_samples or an inconsistent image in the part of the octree the query visits (the
// export's conditions). Reads the ABI only, as the export does, and writes nothing into the context's buffers or Stats.
// Enqueued on the launch stream; returns once complete. *kernel_ms (optional) = event time of the query kernels. Scratch
// memory is the context's (shared with the exports), kept until simlod_destroy.
int simlod_query_region(SimlodContext* ctx, const SimlodRegion* region, int32_t depth, uint64_t dst_samples,
                        uint64_t sample_capacity, SimlodQueryInfo* info, float* kernel_ms);

// Clip volumes (DESIGN.md §9.15): simlod_render and simlod_pick draw only the samples of the LOD cut inside, or outside, a
// union of up to four regions. A sample is `in` when the region query's point predicate (above, on the stored x, y, z)
// holds for at least one of the first num_regions regions. INSIDE draws the samples that are in, OUTSIDE those that are
// not. The clip is context state, kept until it is set again, and changes nothing but which samples of the cut are
// drawn: not the cut, Node::visible / isLarge, Stats, simlod_export_view (pick indices stay indices into it), nor eye-dome
// lighting, the HQS resolve or the overlay, which run on whatever the draw left in the framebuffer.
// SimlodClip {mode SIMLOD_CLIP_*, num_regions, regions[SIMLOD_CLIP_MAX_REGIONS]}: layout in simlod_abi.h.
// clip == NULL or mode SIMLOD_CLIP_NONE: no clip. SIMLOD_ERR_INVALID, with the previous clip left in place, for an unknown
// mode, num_regions 0 (with a mode other than NONE) or above 4, or a region simlod_query_region refuses. Launches nothing.
int simlod_set_clip(SimlodContext* ctx, const SimlodClip* clip);

// Pick (DESIGN.md §9.9): which stored sample each pixel of the frame simlod_render draws for the current uniforms shows, as
// an index into the sample array simlod_export_view returns for the same uniforms (its records say which node holds the
// sample and whether it is a point or a voxel).
typedef struct SimlodPickInfo {
    uint64_t num_hits;                              //   0  requested pixels that show a sample
    uint64_t num_samples;                           //   8  samples of the view export: the index space
    uint32_t num_nodes;                             //  16  records of the view export
    uint32_t num_pixels;                            //  20  pixels requested
    float    plan_ms, key_ms, index_ms, write_ms;   //  24  event time of each stage: the view's plan, the key pass (with
                                                    //      the clear), the index pass, the write
} SimlodPickInfo;
SIMLOD_STATIC_ASSERT(sizeof(SimlodPickInfo) == 40, "PickInfo");
SIMLOD_STATIC_ASSERT(offsetof(SimlodPickInfo, num_nodes) == 16 && offsetof(SimlodPickInfo, plan_ms) == 24, "PickInfo.num_nodes");
//   candidates   every sample S[i] of the view export, projected as kernel_render projects it (pixel (x, y), depth w,
//                inside); a candidate when inside and, with useHighQualityShading, depth > 0. Its key is
//                k = float_bits(depth) << 32 | c, c the colour the frame displays (its own, by node or by level)
//   pixels       a candidate covers clamp(x+ox, 0, W) + W * clamp(y+oy, 0, H) for 0 <= ox, oy < pointSize (W x H the
//                context's frame); ids >= W*H are dropped, an id with x+ox == W wraps into the next row as in the frame
//   winner       of a pixel: the covering candidate with the smallest (k, i). The pixel is hit when k < 0x7f800000_00332211
//                (the frame's clear value), with useHighQualityShading when depth bits < 0x7f800000; never with
//                showPoints == 0. The bounding-box overlay is not part of the result.
// So after simlod_render with the same uniforms (showBoundingBox 0, a cut within the renderer's item capacity), a pixel
// is -1 exactly where the framebuffer holds the clear value, and otherwise the framebuffer holds the winner's key (its
// depth alone with useHighQualityShading) — before eye-dome lighting replaces the colour word of the pixels it shades.
//   pixels == NULL     the whole frame, pixel p = x + W * y at dst_index[p] (num_pixels must be 0)
//   pixels != NULL     num_pixels (x, y) pairs with x < W and y < H, 1 <= num_pixels <= W * H; pixel t at dst_index[t]
// dst_index (int64, 8-byte aligned): the index, or -1. dst_samples (optional, 16-byte aligned): the picked SimlodPoint,
// zeros where the index is -1. Both 0: *info only. SIMLOD_ERR_INVALID before any launch, with nothing written, for a
// pixel outside the frame, an empty or oversized list or a misaligned destination; after the plan, with nothing
// written, for an inconsistent image (the export's conditions). Writes nothing into the context's buffers or Stats
// (not even Node::visible / isLarge); two picks of the same state are byte-identical. Enqueued on the launch stream;
// returns once complete. *kernel_ms (optional) = event time of all its kernels. Scratch: two W x H u64 frames and the
// pixel list, kept until simlod_destroy, besides the export's.
int simlod_pick(SimlodContext* ctx, const uint32_t* pixels, uint64_t num_pixels, uint64_t dst_index, uint64_t dst_samples,
                SimlodPickInfo* info, float* kernel_ms);

// k nearest samples (DESIGN.md §9.10): for each query position, the k samples of a sample set with the smallest key, as
// indices into the sample array simlod_export_octree(depth) returns for the same state (its records say which node holds
// a sample and whether it is a point or a voxel).
#define SIMLOD_NEAREST_MAX_K 32
#define SIMLOD_NEAREST_MAX_QUERIES (1u << 24)
typedef struct SimlodNearestInfo {
    uint64_t num_samples;                           //   0  samples of the export at `depth`: the index space
    uint64_t num_found;                             //   8  filled slots, summed over the queries
    uint64_t samples_tested;                        //  16  distance evaluations, summed over the queries
    uint64_t records_visited;                       //  24  records whose samples were evaluated, summed over the queries
    uint32_t num_queries, k;                        //  32
    uint32_t invalid_queries;                       //  40  queries with a non-finite coordinate (k empty slots each)
    uint32_t max_level;                             //  44  deepest level in the octree
    float    plan_ms, bucket_ms, search_ms;         //  48  event time of the export's plan, of the locate + bucketing, and of
                                                    //      the search (which writes the destinations)
    uint32_t reserved;                              //  60
} SimlodNearestInfo;
SIMLOD_STATIC_ASSERT(sizeof(SimlodNearestInfo) == 64, "NearestInfo");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNearestInfo, num_queries) == 32 && offsetof(SimlodNearestInfo, plan_ms) == 48, "NearestInfo.num_queries");
//   sample set   as simlod_query_region's: depth < 0, the eligible points of every leaf (the inserted point set);
//                0 <= depth <= 20, the export's cut at `depth`, its points eligible ones, its voxels always
//   key          of sample p for query q: d = p - q per coordinate, d2 = (dx*dx + dy*dy) + dz*dz in float32 without
//                contraction (the sphere predicate's sequence); samples are ordered by (d2, index). d2 may be +inf.
//   candidates   the samples of the set with d2 <= max_radius * max_radius (float32); max_radius = +inf for no limit
//   result       k slots per query in ascending key order: dst_index[q][j] (int64), dst_dist2[q][j] (float32) and
//                dst_samples[q][j] (the 16-byte SimlodPoint, bit for bit export_octree(depth).samples[index]). A slot
//                beyond the candidates is empty: index -1, d2 +inf, sample all zero. A query with a non-finite coordinate
//                gets k empty slots and counts in info->invalid_queries.
//   queries      a device address of num_queries 16-byte records (x, y, z, one ignored word), 16-byte aligned, so the
//                samples of an export, a region query or a pick can be passed as they are; queries may lie outside the cube
// Each destination may be 0 (not written). SIMLOD_ERR_INVALID before any launch, with nothing written, for k outside
// 1..SIMLOD_NEAREST_MAX_K, num_queries 0 or above SIMLOD_NEAREST_MAX_QUERIES, depth > 20, a NaN or negative
// max_radius, a null or misaligned query array or a misaligned destination; with nothing written, for an inconsistent
// image (the export's conditions, and a record tree whose levels do not step by one from the root to at most 20). A
// record whose lattice box cannot hold a candidate that beats a query's k-th key is skipped unread, so the result
// equals an exhaustive search, and two calls on the same state are byte-identical. Reads the ABI only, as the export
// does, and writes nothing into the context's buffers or Stats. Enqueued on the launch stream; returns once complete.
// *kernel_ms (optional) = event time of all its kernels. Scratch: the export's, and 12 bytes per query and 12 per record,
// kept until simlod_destroy.
int simlod_query_nearest(SimlodContext* ctx, uint64_t queries, uint64_t num_queries, uint32_t k, int32_t depth, float max_radius,
                         uint64_t dst_index, uint64_t dst_dist2, uint64_t dst_samples, SimlodNearestInfo* info, float* kernel_ms);

// Rays (DESIGN.md §9.11): for each ray, the first sample of a sample set along it within a radius of the ray, as an index
// into the sample array simlod_export_octree(depth) returns for the same state.
#define SIMLOD_RAY_MAX_RAYS (1u << 24)
typedef struct SimlodRayInfo {
    uint64_t num_samples;                           //   0  samples of the export at `depth`: the index space
    uint64_t num_hits;                              //   8  rays with a hit
    uint64_t samples_tested;                        //  16  sample evaluations, summed over the rays
    uint64_t records_visited;                       //  24  records whose samples were evaluated, summed over the rays
    uint32_t num_rays;                              //  32
    uint32_t invalid_rays;                          //  36  rays refused one by one (an empty result each)
    uint32_t max_level;                             //  40  deepest level in the octree
    float    plan_ms, trace_ms;                     //  44  event time of the export's plan, and of the level check and
                                                    //      the trace (which writes the destinations)
    uint32_t reserved;                              //  52
} SimlodRayInfo;
SIMLOD_STATIC_ASSERT(sizeof(SimlodRayInfo) == 56, "RayInfo");
SIMLOD_STATIC_ASSERT(offsetof(SimlodRayInfo, num_rays) == 32 && offsetof(SimlodRayInfo, plan_ms) == 44, "RayInfo.num_rays");
//   rays         a device address of num_rays 32-byte records (ox, oy, oz, tmin, dx, dy, dz, tmax), float32, 16-byte
//                aligned, 1 <= num_rays <= SIMLOD_RAY_MAX_RAYS
//   direction    normalised by the library: len = sqrt((double(dx)*double(dx) + double(dy)*double(dy)) + double(dz)*double(dz)),
//                u = float32(double(d) / len) per axis, every double operation rounded to nearest, nothing contracted
//   invalid ray  an origin or direction that is not finite, a zero direction, tmin NaN, negative or infinite, tmax NaN
//                or below tmin: an empty result, counted in info->invalid_rays (not an error)
//   sample set   as simlod_query_nearest's: depth < 0, the eligible points of every leaf (the inserted point set);
//                0 <= depth <= 20, the export's cut at `depth`, its points eligible ones, its voxels always
//   per sample p float32 without contraction: w = p - o per axis; t = ((wx*ux + wy*uy) + wz*uz) + 0 (the + 0 turns -0
//                into +0); c = w x u (cx = wy*uz - wz*uy, cy = wz*ux - wx*uz, cz = wx*uy - wy*ux);
//                h2 = (cx*cx + cy*cy) + cz*cz. p is a hit when tmin <= t <= tmax and h2 <= radius*radius (float32);
//                a NaN never hits
//   result       per ray the hit with the smallest (t bits, index): dst_index[i] (int64, -1 for none), dst_t[i] (float32,
//                +inf for none), dst_h2[i] (float32, +inf for none), dst_samples[i] (the 16-byte SimlodPoint, bit for bit
//                export_octree(depth).samples[index], zeros for none)
// Each destination may be 0 (not written). SIMLOD_ERR_INVALID before any launch, with nothing written, for a radius that
// is negative or not finite, num_rays 0 or above SIMLOD_RAY_MAX_RAYS, depth > 20, a null or misaligned ray array or a
// misaligned destination; with nothing written, for an inconsistent image (the export's conditions, and a record tree
// whose levels do not step by one from the root to at most 20). A record whose inflated lattice box the ray's segment
// cannot reach before its best hit is skipped unread, so the result equals an exhaustive search, and two calls on the
// same state are byte-identical. Reads the ABI only, as the export does, and writes nothing into the context's buffers
// or Stats. Enqueued on the launch stream; returns once complete. *kernel_ms (optional) = event time of all its kernels.
// Scratch: the export's, and a 40-byte control word, kept until simlod_destroy.
int simlod_query_ray(SimlodContext* ctx, uint64_t rays, uint64_t num_rays, float radius, int32_t depth, uint64_t dst_index,
                     uint64_t dst_t, uint64_t dst_h2, uint64_t dst_samples, SimlodRayInfo* info, float* kernel_ms);

// Fixed-radius neighbourhoods (DESIGN.md §9.12): for each query position, every sample of a sample set within a radius
// of it, in CSR form, as indices into the sample array simlod_export_octree(depth) returns for the same state.
#define SIMLOD_RADIUS_MAX_QUERIES (1u << 24)
typedef struct SimlodRadiusInfo {
    uint64_t num_samples;                           //   0  samples of the export at `depth`: the index space
    uint64_t num_found;                             //   8  neighbours summed over the queries (= offsets[num_queries])
    uint64_t samples_tested;                        //  16  distance evaluations of the count pass, summed over the queries
    uint64_t records_visited;                       //  24  records whose samples were evaluated, summed over the queries
    uint32_t num_queries;                           //  32
    uint32_t invalid_queries;                       //  36  queries with a non-finite coordinate (empty neighbourhood)
    uint32_t max_level;                             //  40  deepest level in the octree
    uint32_t max_found;                             //  44  the largest neighbourhood
    float    plan_ms, bucket_ms, count_ms, write_ms;   //  48  event time of the export's plan, of the locate + bucketing,
                                                    //      of the count pass + the offset scan, and of the write pass
} SimlodRadiusInfo;
SIMLOD_STATIC_ASSERT(sizeof(SimlodRadiusInfo) == 64, "RadiusInfo");
SIMLOD_STATIC_ASSERT(offsetof(SimlodRadiusInfo, num_queries) == 32 && offsetof(SimlodRadiusInfo, plan_ms) == 48, "RadiusInfo.num_queries");
//   sample set   as simlod_query_nearest's: depth < 0, the eligible points of every leaf (the inserted point set);
//                0 <= depth <= 20, the export's cut at `depth`, its points eligible ones, its voxels always
//   neighbour    sample p of query q when d2 <= radius * radius (float32), with d = p - q per coordinate and
//                d2 = (dx*dx + dy*dy) + dz*dz in float32 without contraction (simlod_query_nearest's key). radius must
//                be finite and >= 0; when radius * radius overflows to +inf every sample of the set is a neighbour,
//                including those whose d2 overflowed
//   queries      as simlod_query_nearest's: a device address of num_queries 16-byte records (x, y, z, one ignored
//                word), 16-byte aligned, 1 <= num_queries <= SIMLOD_RADIUS_MAX_QUERIES, so the samples of an export, a
//                region query or a pick can be passed as they are; queries may lie outside the cube. A query with a
//                non-finite coordinate gets an empty neighbourhood and counts in info->invalid_queries
//   result       CSR: dst_offsets (int64, num_queries + 1 entries, offsets[0] = 0); query q's neighbours are
//                [offsets[q], offsets[q+1]) of dst_index (int64 indices into export_octree(depth).samples), dst_dist2
//                (float32 d2) and dst_samples (optional, the 16-byte SimlodPoint, bit for bit the export's sample)
//   order        within a query, the terminal records (records without children) in Z-order: by
//                morton(X, Y, Z at the record's level) << 3 * (20 - level), child index bits x<<2 | y<<1 | z, root
//                first (the record tree's depth-first pre-order with children in octant order); within a record the
//                export's order (points, then voxels). Not ascending index: the export is breadth-first
// dst_index, dst_dist2 and dst_samples all 0: a size query, which fills *info and, when dst_offsets is not 0, the offsets.
// Otherwise `capacity` is the number of neighbour slots of each non-null destination: below info->num_found the call is
// refused with SIMLOD_ERR_INVALID, nothing written into any destination (offsets included) and *info filled. Each of
// dst_index, dst_dist2, dst_samples and dst_offsets may be 0 (not written). SIMLOD_ERR_INVALID before any launch, with
// nothing written, for a radius that is NaN, negative or infinite, num_queries 0 or above SIMLOD_RADIUS_MAX_QUERIES,
// depth > 20, a null or misaligned query array or a misaligned destination (8 / 8 / 4 / 16 bytes); with nothing written,
// for an inconsistent image (the export's conditions, and a record tree whose levels do not step by one from the root
// to at most 20). A record whose lattice box cannot hold a neighbour is skipped unread, so the result equals an
// exhaustive search, and two calls on the same state are byte-identical. Reads the ABI only, as the export does, and
// writes nothing into the context's buffers or Stats. Enqueued on the launch stream; returns once complete.
// *kernel_ms (optional) = event time of all its kernels. Scratch: the export's, simlod_query_nearest's, and 16 bytes per
// query, kept until simlod_destroy.
int simlod_query_radius(SimlodContext* ctx, uint64_t queries, uint64_t num_queries, float radius, int32_t depth,
                        uint64_t dst_offsets, uint64_t dst_index, uint64_t dst_dist2, uint64_t dst_samples,
                        uint64_t capacity, SimlodRadiusInfo* info, float* kernel_ms);

// Height maps (DESIGN.md §9.14): per cell of a grid over the x-y plane, the count, lowest, highest and mean z of the
// samples of a sample set that fall in it, and the highest of them, as an index into the sample array
// simlod_export_octree(depth) returns for the same state.
#define SIMLOD_HEIGHTMAP_MAX_CELLS (1u << 27)
typedef struct SimlodHeightmap {
    float    origin[2];                             //   0  (ox, oy): the low corner of cell (0, 0)
    float    cell;                                  //   8  edge of the square cells
    uint32_t nx, ny;                                //  12  cells per row (x), rows (y)
    uint32_t reserved;                              //  20
} SimlodHeightmap;
SIMLOD_STATIC_ASSERT(sizeof(SimlodHeightmap) == 24, "Heightmap");
SIMLOD_STATIC_ASSERT(offsetof(SimlodHeightmap, cell) == 8 && offsetof(SimlodHeightmap, nx) == 12, "Heightmap.cell");
typedef struct SimlodHeightmapInfo {
    uint64_t num_samples;                           //   0  samples of the export at `depth`: the index space
    uint64_t num_binned;                            //   8  samples that fell in a cell (the sum of the counts)
    uint64_t samples_tested;                        //  16  samples read: those of the chunk items the culling kept
    uint64_t records_visited;                       //  24  records with samples the culling kept
    uint64_t nonempty_cells;                        //  32
    uint32_t max_level;                             //  40  deepest level in the octree
    float    plan_ms, accumulate_ms, finalize_ms;   //  44  event time of the export's plan, of the reset + accumulate,
                                                    //      and of the finalize (which writes the destinations)
} SimlodHeightmapInfo;
SIMLOD_STATIC_ASSERT(sizeof(SimlodHeightmapInfo) == 56, "HeightmapInfo");
SIMLOD_STATIC_ASSERT(offsetof(SimlodHeightmapInfo, max_level) == 40 && offsetof(SimlodHeightmapInfo, plan_ms) == 44, "HeightmapInfo.max_level");
//   grid         cell (i, j) is the square [ox + i cell, ox + (i+1) cell) x [oy + j cell, oy + (j+1) cell) as computed
//                below; results are (ny, nx) arrays, row j, column i, rows in +y order (no image flip)
//   cell of p    in float32, round to nearest, nothing contracted: u = (x - ox) / cell, v = (y - oy) / cell, both IEEE
//                divisions. p counts in cell (trunc(u), trunc(v)) when u >= 0 and v >= 0 (a NaN fails; -0 passes) and
//                trunc(u) < nx, trunc(v) < ny (saturating float -> uint32)
//   sample set   as simlod_query_nearest's: depth < 0, the eligible points of every leaf (the inserted point set);
//                0 <= depth <= 20, the export's cut at `depth`, its points eligible ones, its voxels always
//   z order      the sign-aware bit order of float32 (-0 below +0)
//   result       per cell: dst_count (int64, 0 when empty), dst_z_min, dst_z_max (float32, NaN 0x7fc00000 when empty),
//                dst_z_mean (float32, below), dst_top (int64: the index of the highest sample, equal z to the smallest
//                index; -1 when empty) and dst_samples (the top sample's 16-byte SimlodPoint, bit for bit
//                export_octree(depth).samples[top]; zeros when empty)
//   z_mean       fixed point, in double with every operation rounded to nearest and nothing contracted: size = the cube
//                edge (the largest of boxMax - boxMin in float32), K = 2^30 / size, q = rint_even((z - minz) K) per
//                sample (z, minz = boxMin[2] widened to double), S = the int64 sum of q over the cell, and
//                z_mean = float32(minz + (S / n) / K): the mean of z quantised to 2^-30 of the cube edge
// Each destination may be 0 (not written); with all of them 0 the call fills *info only. SIMLOD_ERR_INVALID before any
// launch, with nothing written, for a null info or grid, a non-finite origin, a cell that is not finite or not > 0, nx
// or ny 0, nx * ny above SIMLOD_HEIGHTMAP_MAX_CELLS (tile larger rasters), depth > 20 or a misaligned destination (8
// bytes for the int64 results, 4 for float32, 16 for samples); after the plan, with nothing written, for an export of
// 2^32 samples or more and for an inconsistent image (the export's conditions). A record whose lattice box cannot hold a
// sample of a cell of the grid is skipped unread, so the result equals binning every sample of the set, and two calls on
// the same state are byte-identical. Reads the ABI only, as the export does, and writes nothing into the context's
// buffers or Stats. Enqueued on the launch stream; returns once complete. *kernel_ms (optional) = event time of all its
// kernels. Scratch: the export's, and up to 24 bytes per cell (4 for the count, 4 for z_min, 8 for z_max / top / samples,
// 8 for z_mean), kept until simlod_destroy.
int simlod_query_heightmap(SimlodContext* ctx, const SimlodHeightmap* grid, int32_t depth, uint64_t dst_count, uint64_t dst_z_min,
                           uint64_t dst_z_max, uint64_t dst_z_mean, uint64_t dst_top, uint64_t dst_samples,
                           SimlodHeightmapInfo* info, float* kernel_ms);

// Octree files (SimlodOctreeFileHeader, DESIGN.md §9.7): a built octree saved and loaded back, so that it can be rendered,
// exported or continued with new batches in another context, process or session.
// simlod_read_octree_header: the header of an octree file, checked against itself and the file size. No context, no GPU.
// SIMLOD_ERR_INVALID, naming the file, for a missing or short file, a wrong magic or version, or section offsets and sizes
// that disagree with the header or the file size.
int simlod_read_octree_header(const char* path, SimlodOctreeFileHeader* out);
// Saves the octree as the last completed kernel_construct left it (batches still waiting in the ring are not part of it):
// the full export's records and samples, the nodes' counters, the box and Stats::batchletIndex / numPointsProcessed.
// Writes nothing into the context's buffers or Stats. SIMLOD_ERR_INVALID for an octree whose Stats::dbg has a bit other
// than SIMLOD_DBG_FAR_POINT set, an inconsistent image, or a file that cannot be written. *info (optional) receives the
// export's counts, *kernel_ms (optional) the event time of the export kernels. Staging memory is bounded (the file
// streamer's page-locked pool and a 256 MB device window), whatever the octree's size.
int simlod_save_octree(SimlodContext* ctx, const char* path, SimlodExportInfo* info, float* kernel_ms);
// Replaces the context's octree by the file's (the counterpart of reload(), like simlod_insert_files): nodes[], heap,
// Stats, the box of the uniforms (camera and settings stay), the ring counters and the builder's side tables, so that the
// next kernel_construct launch continues as it would have in the context that saved the tree. Samples stream through
// the page-locked pool, read by `loader_threads` threads. Errors name the file:
//   SIMLOD_ERR_INVALID  bad header or records that are not a full export: nothing in the context is changed;
//   SIMLOD_ERR_CAPACITY more records than nodes[] holds, more than 65 536 non-empty leaves, or a heap image that does not
//                       fit the persistent buffer below the capacity guard's 200 MB margin: nothing is changed;
//   SIMLOD_ERR_MODULE   a construct program other than the built-in one is loaded: nothing is changed;
//   SIMLOD_ERR_INVALID  found while the samples are placed (a point outside its leaf, a voxel off its cell centre, two
//                       voxels in one cell, a failed read): the context is left reset to an empty octree with the file's box.
int simlod_load_octree(SimlodContext* ctx, const char* path, int loader_threads, SimlodExportInfo* info, float* kernel_ms);

// LAS files written on the GPU (DESIGN.md §9.13): samples quantised and encoded into LAS 1.2 point-format-2 records on
// the device, so that other tools can read what the library holds.
typedef struct SimlodLasWriteParams {
    double scale[3];                                //   0  > 0 and finite
    double offset[3];                               //  24  the file's offset, finite
    double translation[3];                          //  48  added to every sample: world = sample + translation, finite
    uint32_t writer_threads;                        //  72  1..64 threads write the file
    uint32_t reserved;                              //  76
} SimlodLasWriteParams;
SIMLOD_STATIC_ASSERT(sizeof(SimlodLasWriteParams) == 80, "LasWriteParams");
SIMLOD_STATIC_ASSERT(offsetof(SimlodLasWriteParams, translation) == 48 && offsetof(SimlodLasWriteParams, writer_threads) == 72, "LasWriteParams.translation");
typedef struct SimlodLasWriteInfo {
    uint64_t num_points;                            //   0  records written
    uint64_t file_size;                             //   8  227 + 26 * num_points
    uint64_t first_invalid;                         //  16  source index of the first invalid sample, UINT64_MAX for none
    double   min[3];                                //  24  the header's bounds: double(q_min) * scale + offset
    double   max[3];                                //  48      and double(q_max) * scale + offset (0 when empty)
    float    plan_ms;                               //  72  event time of the export's plan + collect (octree source)
    float    encode_ms;                             //  76  event time of the gathers and encodes
    float    copy_ms;                               //  80  event time of the device-to-host copies of the records
    float    write_ms;                              //  84  wall time from the first window to the renamed file
    uint32_t num_windows;                           //  88  windows of at most 8 Mi samples
    uint32_t reserved;                              //  92
} SimlodLasWriteInfo;
SIMLOD_STATIC_ASSERT(sizeof(SimlodLasWriteInfo) == 96, "LasWriteInfo");
SIMLOD_STATIC_ASSERT(offsetof(SimlodLasWriteInfo, min) == 24 && offsetof(SimlodLasWriteInfo, plan_ms) == 72 && offsetof(SimlodLasWriteInfo, num_windows) == 88, "LasWriteInfo.min");
//   source       samples != 0: num_samples 16-byte samples (x, y, z, colour bits) at that 16-byte aligned device address,
//                depth < 0 (the layout of export_*, query_region and the queries' samples). samples == 0: the octree's
//                samples as the last completed launch left it, depth < 0 the inserted points (the export's cut at 20,
//                the points on the cube's max face included), 0 <= depth <= 20 the export's cut at depth; num_samples
//                is then ignored. Record i of the file is sample i of the source (export_octree(depth).samples, with
//                depth 20 for depth < 0).
//   quantised    per axis in IEEE double, nothing contracted: q = rint(((double(p) + translation) - offset) / scale),
//                half to even. A sample with a non-finite coordinate or a q outside int32 is invalid.
//   file         LAS 1.2, 227-byte header, no VLRs, point format 2 (26 bytes: int32 X, Y, Z = q, intensity 0, flags
//                0x09, classification, scan angle, user data and point source 0, R, G, B = 257 * colour bits 0-7,
//                8-15, 16-23); generating software "simlod_b200", creation day and year 0; legacy point count n and
//                points by return [n, 0, 0, 0, 0]; scale and offset as given; min / max as in SimlodLasWriteInfo.
// SIMLOD_ERR_INVALID before any launch, with no file created, for a null path, params or info, a scale that is not
// finite or <= 0, a non-finite offset or translation, a misaligned samples address, samples != 0 with depth >= 0,
// depth > 20, more than 2^32 - 1 samples of the caller's, writer_threads outside 1..64, or a path whose directory
// cannot be written. SIMLOD_ERR_INVALID during the write for an invalid sample (info->first_invalid names the first one
// in source order), more than 2^32 - 1 samples of the octree's, an inconsistent image or an I/O error. The file is
// written as path + ".tmp" and renamed once complete: a failed call leaves no file and any existing file at `path` as
// it was. Writes nothing into the context's buffers or Stats. *kernel_ms (optional) = event time of all its kernels.
// Staging: the file streamer's page-locked pool, and a 208 MiB device window (plus the octree file's sample window for
// the octree source), kept until simlod_destroy.
int simlod_write_las(SimlodContext* ctx, const char* path, const SimlodLasWriteParams* params, uint64_t samples,
                     uint64_t num_samples, int32_t depth, SimlodLasWriteInfo* info, float* kernel_ms);
// The union box of a list of .las / .simlod files as simlod_insert_files computes it (float header bounds), with the
// same validation and errors; an octree built from the list holds its points at (world - box_min). No context, no GPU.
int simlod_files_box(const char* const* paths, uint32_t num_paths, float box_min[3], float box_max[3]);

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
