// kernel_args.h — the argument and control structs that host.cpp fills and the kernels read, with the codes and limits
// both sides use. One definition for both compilers: plain C++ (no device code), included by host.cpp and by export.cu,
// query.cu, pick.cu, nearest.cu, radius.cu, ray.cu and heightmap.cu (through export_common.cuh), import.cu, partition.cu and las_write.cu. The static_asserts pin
// every size, and the offsets that one side reads of a struct the other writes, so a layout change fails to compile instead
// of shifting bytes.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/simlod_abi.h"

// ---- octree export (export.cu) and region query (query.cu) ---------------------------------------------------------

enum : uint32_t {                         // ExportCtl::error (the canonicaliser's codes, oracle.cpp canonFromImage)
    EXPORT_ERR_CHILD = 1,                 // a child pointer outside nodes[] (or more records than nodes: a node reached twice)
    EXPORT_ERR_CHUNK = 2,                 // a chunk pointer outside the used heap
    EXPORT_ERR_SHORT = 4,                 // a list shorter than its count
    EXPORT_ERR_PARTIAL = 5,               // an inner node without all 8 children
};

struct ExportCtl {                        // the plan's sizes and error, read back by the host before the gather
    uint32_t numNodes, maxLevel;
    uint64_t numSamples, numPoints, numVoxels;
    uint64_t numItems;
    uint32_t error, pad;
};
static_assert(sizeof(ExportCtl) == 48 && offsetof(ExportCtl, numItems) == 32 && offsetof(ExportCtl, error) == 40, "ExportCtl");

// The view export's scratch (all null for the full and depth exports). The breadth-first pass writes the record of every
// reachable node into rec / recNode here; the records the view keeps are then compacted into the plan's rec / recNode.
struct ViewScratch {
    const uint8_t* drawn;         // [node index] 1 when kernel_render draws the node (simlod_export_view_flags)
    SimlodExportNode* rec;        // [record] breadth-first records of every reachable node
    uint32_t* recNode;            // [record] their node indices
    uint8_t* mark;                // [record] 1 when a drawn record lies strictly below
    uint32_t* index;              // [record] position among the kept records
};
static_assert(sizeof(ViewScratch) == 40, "ViewScratch");

struct QueryCtl {                         // simlod_export_collect sees the ExportCtl it begins with
    ExportCtl plan;                       // records, candidate samples (those of the visited nodes), items, error
    uint64_t outSamples, outPoints, outVoxels;
    uint32_t nodesVisited, pad;
};
static_assert(sizeof(QueryCtl) == 80 && offsetof(QueryCtl, plan) == 0 && offsetof(QueryCtl, outSamples) == 48, "QueryCtl");

struct QueryBox { float mn[3], mx[3]; };  // boxMin / boxMax of the uniforms
static_assert(sizeof(QueryBox) == 24, "QueryBox");

// ---- pick (pick.cu) -------------------------------------------------------------------------------------------------

struct PickArgs {                         // the view export's plan (export scratch) and the pick's two frames
    const SimlodExportNode* rec;          // [record] the view's records
    const uint64_t* recItem;              // [record] its first chunk item
    const uint64_t* items;                // [item] two words: Item {src, dst | count << 48} (export_common.cuh)
    uint64_t* key;                        // [pixel] smallest candidate key depth << 32 | colour
    uint64_t* index;                      // [pixel] smallest sample index with that key, ~0 for none
    uint64_t* hits;                       // picked pixels among those the write kernel visits
    uint64_t numItems;
    uint32_t numRecords, pad;
    SimlodClip clip;                      // the context's clip: candidates are the samples it keeps (mode NONE: all)
};
static_assert(sizeof(PickArgs) == 1288 && offsetof(PickArgs, numItems) == 48 && offsetof(PickArgs, clip) == 64, "PickArgs");

// ---- k nearest samples (nearest.cu) ----------------------------------------------------------------------------------

constexpr uint32_t NEAREST_RUN = 8;       // queries per block of the search, one warp each

struct NearestCtl {                       // zeroed by the host before the locate; read back after the search
    uint32_t error;                       // EXPORT_ERR_CHILD: a record tree deeper than 20 levels or with levels out of step
    uint32_t numRuns;                     // blocks the search needs: runs of up to NEAREST_RUN queries with one home
    uint64_t numFound, samplesTested, recordsVisited, invalid;
};
static_assert(sizeof(NearestCtl) == 40 && offsetof(NearestCtl, numFound) == 8, "NearestCtl");

struct NearestArgs {                      // the export's plan (export scratch), the query's scratch and its destinations
    const SimlodExportNode* rec;          // [record] the plan's breadth-first records
    const uint64_t* recItem;              // [record] first chunk item of the record's point list (its voxel list follows)
    const uint64_t* items;                // [item] two words: Item {src, dst | count << 48} (export_common.cuh)
    const float* queries;                 // [query] 16-byte records x, y, z, ignored
    uint32_t* home;                       // [query] home record; numRecords for a query with a non-finite coordinate
    uint32_t* slot;                       // [query] position in its home's bucket
    uint32_t* count;                      // [home] queries per home record (numRecords + 1 homes)
    uint32_t* offset;                     // [home] first bucket position of the home
    uint32_t* runStart;                   // [home] first run of the home; [numRecords + 1] = the number of runs
    uint32_t* bucket;                     // [position] query ids grouped by home
    NearestCtl* ctl;
    int64_t* dstIndex;                    // [query][k] or null
    float* dstDist2;                      // [query][k] or null
    SimlodPoint* dstSamples;              // [query][k] or null
    uint32_t numQueries, numRecords, k;
    int32_t depth;                        // < 0: the points of the leaves; else the export's cut at `depth`
    float maxRadius;
    float boxMin[3], boxMax[3];           // of the uniforms: the octree cube
    uint32_t pad;
};
static_assert(sizeof(NearestArgs) == 160 && offsetof(NearestArgs, numQueries) == 112 && offsetof(NearestArgs, boxMin) == 132, "NearestArgs");

// ---- fixed-radius neighbourhoods (radius.cu, after nearest.cu's locate, scan and scatter) ----------------------------

constexpr uint32_t RADIUS_SCAN_ITEMS = 8;                       // counts per thread of the offset scan
constexpr uint32_t RADIUS_SCAN_TILE = 1024 * RADIUS_SCAN_ITEMS; // counts per block of the offset scan

struct RadiusCtl {                        // zeroed by the host before the locate; read back after the scan
    uint64_t numFound, samplesTested, recordsVisited, invalid;   // summed by the count pass
    uint32_t maxFound, pad;
};
static_assert(sizeof(RadiusCtl) == 40 && offsetof(RadiusCtl, maxFound) == 32, "RadiusCtl");

struct RadiusArgs {                       // the export's plan (export scratch), nearest.cu's buckets, the pass scratch and
                                          // the destinations
    const SimlodExportNode* rec;          // [record] the plan's breadth-first records
    const uint64_t* recItem;              // [record] first chunk item of the record's point list (its voxel list follows)
    const uint64_t* items;                // [item] two words: Item {src, dst | count << 48} (export_common.cuh)
    const float* queries;                 // [query] 16-byte records x, y, z, ignored
    const uint32_t* count;                // [home] queries per home record (numRecords + 1 homes), from the locate
    const uint32_t* offset;               // [home] first bucket position of the home
    const uint32_t* runStart;             // [home] first run of the home; [numRecords + 1] = the number of runs
    const uint32_t* bucket;               // [position] query ids grouped by home
    const NearestCtl* nearestCtl;         // the scan's error and number of runs
    RadiusCtl* ctl;
    uint32_t* total;                      // [query] neighbours
    uint32_t* before;                     // [query] neighbours in terminal records before the home in Z-order
    uint64_t* tileSum;                    // [scan tile] sum of its totals
    int64_t* offsets;                     // [query + 1] exclusive prefix of the totals
    int64_t* dstIndex;                    // [neighbour] or null
    float* dstDist2;                      // [neighbour] or null
    SimlodPoint* dstSamples;              // [neighbour] or null
    uint32_t numQueries, numRecords;
    int32_t depth;                        // < 0: the points of the leaves; else the export's cut at `depth`
    float radius;
    float boxMin[3], boxMax[3];           // of the uniforms: the octree cube
};
static_assert(sizeof(RadiusArgs) == 176 && offsetof(RadiusArgs, numQueries) == 136 && offsetof(RadiusArgs, boxMin) == 152, "RadiusArgs");

// ---- rays (ray.cu) ---------------------------------------------------------------------------------------------------

constexpr uint32_t RAY_WARPS = 8;         // rays per block of the trace, one warp each

struct RayCtl {                           // zeroed by the host before the check; read back after the trace
    uint32_t error;                       // EXPORT_ERR_CHILD: a record tree deeper than 20 levels or with levels out of step
    uint32_t pad;
    uint64_t numHits, samplesTested, recordsVisited, invalid;
};
static_assert(sizeof(RayCtl) == 40 && offsetof(RayCtl, numHits) == 8, "RayCtl");

struct RayArgs {                          // the export's plan (export scratch), the rays and the destinations
    const SimlodExportNode* rec;          // [record] the plan's breadth-first records
    const uint64_t* recItem;              // [record] first chunk item of the record's point list (its voxel list follows)
    const uint64_t* items;                // [item] two words: Item {src, dst | count << 48} (export_common.cuh)
    const float* rays;                    // [ray] 32-byte records ox, oy, oz, tmin, dx, dy, dz, tmax
    RayCtl* ctl;
    int64_t* dstIndex;                    // [ray] or null
    float* dstT;                          // [ray] or null
    float* dstH2;                         // [ray] or null
    SimlodPoint* dstSamples;              // [ray] or null
    uint32_t numRays, numRecords;
    int32_t depth;                        // < 0: the points of the leaves; else the export's cut at `depth`
    float radius;
    float boxMin[3], boxMax[3];           // of the uniforms: the octree cube
};
static_assert(sizeof(RayArgs) == 112 && offsetof(RayArgs, numRays) == 72 && offsetof(RayArgs, boxMin) == 88, "RayArgs");

// ---- height maps (heightmap.cu) --------------------------------------------------------------------------------------

struct HeightmapCtl {                     // zeroed by the host before the accumulate; read back after the finalize
    uint64_t numBinned, samplesTested, recordsVisited;   // summed by the accumulate, in this order
    uint64_t nonemptyCells;               // summed by the finalize
};
static_assert(sizeof(HeightmapCtl) == 32 && offsetof(HeightmapCtl, nonemptyCells) == 24, "HeightmapCtl");

struct HeightmapArgs {                    // the export's plan (export scratch), the per-cell accumulators and the destinations
    const SimlodExportNode* rec;          // [record] the plan's breadth-first records
    const uint64_t* recItem;              // [record] first chunk item of the record's point list (its voxel list follows)
    const uint64_t* items;                // [item] two words: Item {src, dst | count << 48} (export_common.cuh)
    HeightmapCtl* ctl;
    uint32_t* count;                      // [cell] binned samples (memset 0)
    uint32_t* zmin;                       // [cell] the least ordered z (memset 0xff), or null when not needed
    unsigned long long* top;              // [cell] ordered(z) << 32 | (0xffffffff - index), the largest (memset 0), or null
    unsigned long long* sum;              // [cell] the sum of the fixed-point z (memset 0), or null
    int64_t* dstCount;                    // [cell] or null
    float* dstZMin;                       // [cell] or null
    float* dstZMax;                       // [cell] or null
    float* dstZMean;                      // [cell] or null
    int64_t* dstTop;                      // [cell] or null
    SimlodPoint* dstSamples;              // [cell] or null
    uint64_t numItems;
    uint32_t numRecords;
    int32_t depth;                        // < 0: the points of the leaves; else the export's cut at `depth`
    uint32_t nx, ny;                      // cells per row, rows
    float origin[2], cell;
    float boxMin[3], boxMax[3];           // of the uniforms: the octree cube
    uint32_t pad;
};
static_assert(sizeof(HeightmapArgs) == 176 && offsetof(HeightmapArgs, numItems) == 112 && offsetof(HeightmapArgs, origin) == 136 &&
              offsetof(HeightmapArgs, boxMin) == 148, "HeightmapArgs");

// ---- LAS writer (las_write.cu) ---------------------------------------------------------------------------------------

constexpr uint32_t LAS_WRITE_TILE = 256;                        // samples per block iteration of the encode
constexpr uint32_t LAS_WRITE_RECORD = 26;                       // bytes of a point-format-2 record
constexpr uint64_t LAS_WRITE_WINDOW = 8ull << 20;               // samples per window (208 MiB of records)

// Every word is an unsigned minimum, so that one memset of 0xff resets the whole struct once per call: qmin holds
// q ^ 0x80000000 (signed order as unsigned), qmaxInv holds ~(q ^ 0x80000000). Read back with each window's records.
struct LasWriteCtl {
    uint32_t qmin[3], qmaxInv[3];         // over the valid samples of every window encoded so far
    uint64_t firstInvalid;                // source index of the first invalid sample, UINT64_MAX for none
    uint64_t pad;
};
static_assert(sizeof(LasWriteCtl) == 40 && offsetof(LasWriteCtl, firstInvalid) == 24, "LasWriteCtl");

struct LasEncodeArgs {
    const SimlodPoint* samples;           // [i] the window's samples, 16-byte aligned
    uint8_t* records;                     // [i] their 26-byte records, 16-byte aligned
    LasWriteCtl* ctl;
    uint64_t first;                       // source index of samples[0]
    uint64_t count;                       // samples in the window
    double scale[3], offset[3], translation[3];
};
static_assert(sizeof(LasEncodeArgs) == 112 && offsetof(LasEncodeArgs, scale) == 40 && offsetof(LasEncodeArgs, translation) == 88, "LasEncodeArgs");

// ---- octree import (import.cu) ------------------------------------------------------------------------------------

enum : uint32_t {                         // the import's error word
    IMPORT_ERR_POINT = 1,                 // a point whose descent does not end in its leaf
    IMPORT_ERR_VOXEL = 2,                 // a voxel that is not the centre of a cell of its node
    IMPORT_ERR_DUPLICATE = 4,             // two voxels in one cell of a node
    IMPORT_ERR_COUNT = 8,                 // a node's voxels are not as many as the cells its points occupy
};

struct ImportPlan {                       // per record; one more entry after the last record (chunk = total)
    uint64_t grid;                        // heap offset of the node's grid (0: none)
    uint64_t chunk;                       // index of its first chunk: points first, then voxels
    uint32_t row;                         // its chunk row (+1; 0: none)
    uint32_t counter;                     // Node::counter from the file
};
static_assert(sizeof(ImportPlan) == 24, "ImportPlan");

struct ImportArgs {
    SimlodNode* nodes;
    uint8_t* heap;
    uint8_t* scratch;                     // kernel_construct's momentary buffer
    const SimlodExportNode* rec;
    const ImportPlan* plan;
    uint32_t* error;
    uint64_t chunkBase;                   // heap offset of chunk 0
    uint32_t numRecords, numRows;
    float boxMin[3], boxMax[3];
};
static_assert(sizeof(ImportArgs) == 88 && offsetof(ImportArgs, chunkBase) == 48 && offsetof(ImportArgs, boxMin) == 64, "ImportArgs");

// ---- spatial exchange and depth compositing (partition.cu) --------------------------------------------------------

namespace part {
constexpr uint32_t MAX_RANKS = 8;
constexpr uint32_t MAX_CELLS = 512;       // level <= 3
constexpr uint32_t BLOCK = 256;           // threads per block of every partition kernel
}  // namespace part

struct PartitionParams {
    float minx, miny, minz, size;           // octree cube: boxMin + max extent (voxels.cu:860-863)
    uint32_t level;                         // 1..3
    uint32_t numRanks;                      // 1..8
    uint32_t count;
    uint32_t perBlock;                      // points per block, a multiple of BLOCK
    uint8_t owner[part::MAX_CELLS];         // cell (Morton order: child index per level, root first) -> rank
};
static_assert(sizeof(PartitionParams) == 544 && offsetof(PartitionParams, owner) == 32, "PartitionParams");

struct ScatterTargets {
    uint64_t ptr[part::MAX_RANKS];          // destination buffers (device addresses, local or peer)
    uint64_t offset[part::MAX_RANKS];       // first point slot of THIS sender in each destination
    uint64_t signal[part::MAX_RANKS];       // this sender's flag word in each destination (0 = no signalling)
    uint32_t signalValue;
    uint32_t pad;
};
static_assert(sizeof(ScatterTargets) == 200 && offsetof(ScatterTargets, signalValue) == 192, "ScatterTargets");

struct CompositeArgs {
    uint64_t fb[part::MAX_RANKS];           // every rank's framebuffer copy (device addresses, local or peer)
    uint64_t signal[part::MAX_RANKS];
    uint64_t numWords;
    uint32_t numRanks, rank, signalValue, pad;
};
static_assert(sizeof(CompositeArgs) == 152 && offsetof(CompositeArgs, numWords) == 128, "CompositeArgs");

struct SignalArgs { uint64_t signal[part::MAX_RANKS]; uint32_t numRanks, value; };
static_assert(sizeof(SignalArgs) == 72 && offsetof(SignalArgs, numRanks) == 64, "SignalArgs");
