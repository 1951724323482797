// simlod_abi.h — host/device ABI of the SimLOD hot path, restated byte-for-byte.
//
// These are the structs that cross the reference's launch boundary. The layouts are
// re-declared here (not copied) and every size/offset that the reference's kernels and
// host rely on is pinned with a static_assert, so that our kernels can be launched by
// the reference host (modules/progressive_octree/main_progressive_octree.cpp:333-546)
// and the reference kernels can be launched by our host, on the same buffers.
//
//   Point          modules/progressive_octree/structures.cuh:30-35   (16 B)
//   Chunk          modules/progressive_octree/structures.cuh:62-67   (16016 B, heap stride 16032)
//   OccupancyGrid  modules/progressive_octree/structures.cuh:69-72   (262144 B, heap stride 262160)
//   Node           modules/progressive_octree/structures.cuh:74-144  (152 B)
//   Uniforms/Stats modules/progressive_octree/HostDeviceInterface.h:10-71 (480 B / 112 B)
//   constants      modules/progressive_octree/structures.cuh:21-28
#pragma once
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
#define SIMLOD_STATIC_ASSERT(c, m) static_assert(c, m)
#else
#define SIMLOD_STATIC_ASSERT(c, m) _Static_assert(c, m)
#endif

enum {
    SIMLOD_MAX_POINTS_PER_NODE = 50000,     // leaf capacity, inclusive (structures.cuh:21, voxels.cu:211-212)
    SIMLOD_POINTS_PER_CHUNK    = 1000,      // structures.cuh:22
    SIMLOD_GRID_SIZE           = 128,       // structures.cuh:23
    SIMLOD_GRID_WORDS          = 128 * 128 * 128 / 32,
    SIMLOD_MAX_DEPTH           = 20,        // structures.cuh:25
    SIMLOD_BATCH_STREAM_SIZE   = 50,        // ring slots (structures.cuh:28, main.cpp:36)
    SIMLOD_MAX_BATCH_SIZE      = 1000000,   // points per ring slot (main.cpp:37)
    SIMLOD_CHUNK_STRIDE        = 16032,     // 16*((16016+16)/16)   (utils.h.cu:185-197)
    SIMLOD_GRID_STRIDE         = 262160,    // 16*((262144+16)/16)
};

typedef struct SimlodPoint {
    float    x, y, z;
    uint32_t color;   // 0xAABBGGRR
} SimlodPoint;

typedef struct SimlodChunk {
    SimlodPoint        points[SIMLOD_POINTS_PER_CHUNK];
    int32_t            size;        // never written by the reference
    int32_t            padding_0;
    struct SimlodChunk* next;
} SimlodChunk;

typedef struct SimlodOccupancyGrid {
    uint32_t values[SIMLOD_GRID_WORDS];   // bit index = x + 128*y + 128*128*z
} SimlodOccupancyGrid;

typedef struct SimlodNode {
    struct SimlodNode*   children[8];   //   0  child index = x<<2 | y<<1 | z
    uint32_t             counter;       //  64  points ever counted into this node while it was a leaf
    uint32_t             numPoints;     //  68  points stored in `points`
    uint32_t             level;         //  72
    uint32_t             X, Y, Z;       //  76  node coordinate at `level`
    uint32_t             countIteration;//  88
    uint32_t             countFlag;     //  92
    uint8_t              name[20];      //  96  'r' + one digit per level
    uint8_t              visible;       // 116  written by kernel_render
    uint8_t              isFiltered;    // 117
    uint8_t              isLeaf;        // 118  stays 1 forever in the reference (never updated)
    uint8_t              isLarge;       // 119  written by kernel_render
    SimlodOccupancyGrid* grid;          // 120
    SimlodChunk*         points;        // 128
    SimlodChunk*         voxelChunks;   // 136
    uint32_t             numVoxels;     // 144
    uint32_t             numVoxelsStored;//148
} SimlodNode;

typedef struct SimlodFloat4 { float x, y, z, w; } SimlodFloat4;
typedef struct SimlodMat4   { SimlodFloat4 rows[4]; } SimlodMat4;   // HostDeviceInterface.h:6-8 (row-major: host stores glm::transpose)

typedef struct SimlodUniforms {
    float      width;                      //   0
    float      height;                     //   4
    float      time;                       //   8
    float      fovy_rad;                   //  12
    SimlodMat4 world;                      //  16
    SimlodMat4 view;                       //  80
    SimlodMat4 proj;                       // 144
    SimlodMat4 transform;                  // 208
    SimlodMat4 transform_updateBound;      // 272
    SimlodMat4 transformInv_updateBound;   // 336
    uint64_t   persistentBufferCapacity;   // 400
    uint64_t   momentaryBufferCapacity;    // 408
    uint64_t   frameCounter;               // 416
    float      boxMin[3];                  // 424
    float      boxMax[3];                  // 436
    uint8_t    showBoundingBox;            // 448 nonzero: kernel_render draws, after the samples and before EDL, the
                                           //     frustum of transformInv_updateBound (8 lines, colour 0x000000ff) and
                                           //     the box of every drawn node (12 lines, 0x0000ff00), 1-pixel lines
                                           //     clipped to and projected by `transform`, depth-tested by atomicMin
                                           //     (the reference's frame; above 10 416 drawn nodes, where the reference
                                           //     overruns its line list, every box is still drawn)
    uint8_t    showPoints;                 // 449
    uint8_t    colorByNode;                // 450
    uint8_t    colorByLOD;                 // 451
    uint8_t    colorWhite;                 // 452
    uint8_t    doUpdateVisibility;         // 453
    uint8_t    doProgressive;              // 454
    uint8_t    _pad0;
    float      LOD;                        // 456
    uint8_t    useHighQualityShading;      // 460
    uint8_t    _pad1[3];
    float      minNodeSize;                // 464
    int32_t    pointSize;                  // 468
    uint8_t    updateStats;                // 472
    uint8_t    enableEDL;                  // 473
    uint8_t    _pad2[2];
    float      edlStrength;                // 476
} SimlodUniforms;

typedef struct SimlodStats {
    uint32_t frameID;                     //   0
    uint32_t numNodes;                    //   4  allocation cursor into nodes[] (1 after reset, +8 per split)
    uint32_t numInner;                    //   8
    uint32_t numLeaves;                   //  12
    uint32_t numNonemptyLeaves;           //  16
    uint32_t numPoints;                   //  20
    uint32_t numVoxels;                   //  24
    uint32_t _pad0;
    uint64_t allocatedBytes_momentary;    //  32
    uint64_t allocatedBytes_persistent;   //  40
    uint32_t numVisibleNodes;             //  48
    uint32_t numVisibleInner;             //  52
    uint32_t numVisibleLeaves;            //  56
    uint32_t numVisiblePoints;            //  60
    uint32_t numVisibleVoxels;            //  64
    uint32_t numChunksPoints;             //  68
    uint32_t numChunksVoxels;             //  72
    uint32_t batchletIndex;               //  76
    uint64_t numPointsProcessed;          //  80
    uint64_t numAllocatedChunks;          //  88
    uint64_t chunkPoolSize;               //  96
    uint32_t dbg;                         // 104
    uint8_t  memCapacityReached;          // 108
    uint8_t  _pad1[3];
} SimlodStats;

// header of the persistent heap (utils.h.cu:180-227, reset.cu:40-43): lives at heap byte 0
typedef struct SimlodHeapHeader {
    uint8_t* buffer;
    uint64_t offset;    // starts at 16; every alloc advances by 16*((size+16)/16)
} SimlodHeapHeader;

// One node of an exported octree (simlod_export_octree). Records are in breadth-first order: by level, then by the
// Morton code of (X, Y, Z) with bit triples x<<2 | y<<1 | z (the child index), so the 8 children of a node are
// consecutive records.
enum {
    SIMLOD_EXPORT_LEAF    = 1u << 0,   // the node has no children
    SIMLOD_EXPORT_SAMPLED = 1u << 1,   // the node's samples are part of this export
};
typedef struct SimlodExportNode {
    uint32_t level, X, Y, Z;           //  0  as in Node
    uint8_t  name[20];                 // 16  as in Node
    uint32_t flags;                    // 36  SIMLOD_EXPORT_*
    int32_t  parent;                   // 40  record index, -1 for the root
    int32_t  first_child;              // 44  record index of child 0, -1 if it has no children or they are not exported
    uint64_t sample_offset;            // 48  index of its first sample in the sample array
    uint32_t num_points;               // 56  exported points, stored first
    uint32_t num_voxels;               // 60  exported voxels, stored right after the points
} SimlodExportNode;

typedef struct SimlodExportInfo {
    uint32_t num_nodes, max_level;     // records in this export; deepest level in the octree
    uint64_t num_samples, num_points, num_voxels;
} SimlodExportInfo;

// Header of an octree file (simlod_save_octree / simlod_load_octree), format version 1, little-endian. The file is this
// 128-byte header, then `info.num_nodes` SimlodExportNode records (byte for byte the node table of the full export), then
// one u32 Node::counter per record, then, at a 16-byte aligned offset, `info.num_samples` 16-byte samples (byte for byte
// the full export's sample array). Reserved bytes are zero.
#define SIMLOD_OCTREE_MAGIC "SIMLODOT"
enum { SIMLOD_OCTREE_VERSION = 1, SIMLOD_OCTREE_HEADER_SIZE = 128 };
typedef struct SimlodOctreeFileHeader {
    char             magic[8];             //   0  "SIMLODOT", no terminator
    uint32_t         version;              //   8  SIMLOD_OCTREE_VERSION
    uint32_t         header_size;          //  12  SIMLOD_OCTREE_HEADER_SIZE
    SimlodExportInfo info;                 //  16  the full export's counts and deepest level
    float            box_min[3];           //  48  Uniforms::boxMin at save time
    float            box_max[3];           //  60  Uniforms::boxMax at save time
    uint32_t         batchlet_index;       //  72  Stats::batchletIndex
    uint32_t         reserved0;            //  76
    uint64_t         num_points_processed; //  80  Stats::numPointsProcessed
    uint64_t         records_offset;       //  88  = header_size
    uint64_t         counters_offset;      //  96  = records_offset + 64 * num_nodes
    uint64_t         samples_offset;       // 104  = counters_offset + 4 * num_nodes, rounded up to 16
    uint64_t         file_size;            // 112  = samples_offset + 16 * num_samples
    uint64_t         reserved1;            // 120
} SimlodOctreeFileHeader;

// The LAS public header fields the reference reads (LasLoader.h:21-55), at their file byte offsets:
typedef struct SimlodLasHeader {
    uint32_t version_major, version_minor;        // bytes 24, 25 (u8)
    uint32_t format, bytes_per_point;             // 104 (u8), 105 (u16)
    uint32_t header_size, offset_to_point_data;   // 94 (u16), 96 (u32)
    uint64_t num_points;                          // 107 (u32) for versions 1.0-1.3, else 247 (u64)
    double   scale[3], offset[3];                 // 131, 155
    double   min[3], max[3];                      // min 187 / 203 / 219, max 179 / 195 / 211
} SimlodLasHeader;

SIMLOD_STATIC_ASSERT(sizeof(SimlodPoint) == 16, "Point");
SIMLOD_STATIC_ASSERT(sizeof(SimlodChunk) == 16016, "Chunk");
SIMLOD_STATIC_ASSERT(offsetof(SimlodChunk, size) == 16000, "Chunk.size");
SIMLOD_STATIC_ASSERT(offsetof(SimlodChunk, next) == 16008, "Chunk.next");
SIMLOD_STATIC_ASSERT(sizeof(SimlodOccupancyGrid) == 262144, "OccupancyGrid");
SIMLOD_STATIC_ASSERT(sizeof(SimlodNode) == 152, "Node");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, counter) == 64, "Node.counter");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, numPoints) == 68, "Node.numPoints");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, level) == 72, "Node.level");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, X) == 76, "Node.X");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, countIteration) == 88, "Node.countIteration");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, name) == 96, "Node.name");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, visible) == 116, "Node.visible");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, isLarge) == 119, "Node.isLarge");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, grid) == 120, "Node.grid");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, points) == 128, "Node.points");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, voxelChunks) == 136, "Node.voxelChunks");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, numVoxels) == 144, "Node.numVoxels");
SIMLOD_STATIC_ASSERT(offsetof(SimlodNode, numVoxelsStored) == 148, "Node.numVoxelsStored");
SIMLOD_STATIC_ASSERT(sizeof(SimlodUniforms) == 480, "Uniforms");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, transform) == 208, "Uniforms.transform");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, transform_updateBound) == 272, "Uniforms.transform_updateBound");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, persistentBufferCapacity) == 400, "Uniforms.persistentBufferCapacity");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, boxMin) == 424, "Uniforms.boxMin");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, boxMax) == 436, "Uniforms.boxMax");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, showBoundingBox) == 448, "Uniforms.showBoundingBox");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, LOD) == 456, "Uniforms.LOD");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, useHighQualityShading) == 460, "Uniforms.useHighQualityShading");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, minNodeSize) == 464, "Uniforms.minNodeSize");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, pointSize) == 468, "Uniforms.pointSize");
SIMLOD_STATIC_ASSERT(offsetof(SimlodUniforms, edlStrength) == 476, "Uniforms.edlStrength");
SIMLOD_STATIC_ASSERT(sizeof(SimlodStats) == 112, "Stats");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, numNodes) == 4, "Stats.numNodes");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, allocatedBytes_momentary) == 32, "Stats.allocatedBytes_momentary");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, numVisibleNodes) == 48, "Stats.numVisibleNodes");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, batchletIndex) == 76, "Stats.batchletIndex");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, numPointsProcessed) == 80, "Stats.numPointsProcessed");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, numAllocatedChunks) == 88, "Stats.numAllocatedChunks");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, chunkPoolSize) == 96, "Stats.chunkPoolSize");
SIMLOD_STATIC_ASSERT(offsetof(SimlodStats, memCapacityReached) == 108, "Stats.memCapacityReached");
SIMLOD_STATIC_ASSERT(sizeof(SimlodExportNode) == 64, "ExportNode");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportNode, name) == 16, "ExportNode.name");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportNode, flags) == 36, "ExportNode.flags");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportNode, parent) == 40, "ExportNode.parent");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportNode, first_child) == 44, "ExportNode.first_child");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportNode, sample_offset) == 48, "ExportNode.sample_offset");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportNode, num_points) == 56, "ExportNode.num_points");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportNode, num_voxels) == 60, "ExportNode.num_voxels");
SIMLOD_STATIC_ASSERT(sizeof(SimlodExportInfo) == 32, "ExportInfo");
SIMLOD_STATIC_ASSERT(sizeof(SimlodLasHeader) == 128, "LasHeader");
SIMLOD_STATIC_ASSERT(offsetof(SimlodLasHeader, num_points) == 24, "LasHeader.num_points");
SIMLOD_STATIC_ASSERT(offsetof(SimlodLasHeader, scale) == 32, "LasHeader.scale");
SIMLOD_STATIC_ASSERT(offsetof(SimlodLasHeader, min) == 80, "LasHeader.min");
SIMLOD_STATIC_ASSERT(offsetof(SimlodLasHeader, max) == 104, "LasHeader.max");
SIMLOD_STATIC_ASSERT(offsetof(SimlodExportInfo, num_samples) == 8, "ExportInfo.num_samples");
SIMLOD_STATIC_ASSERT(sizeof(SimlodOctreeFileHeader) == 128, "OctreeFileHeader");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, version) == 8, "OctreeFileHeader.version");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, header_size) == 12, "OctreeFileHeader.header_size");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, info) == 16, "OctreeFileHeader.info");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, box_min) == 48, "OctreeFileHeader.box_min");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, box_max) == 60, "OctreeFileHeader.box_max");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, batchlet_index) == 72, "OctreeFileHeader.batchlet_index");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, num_points_processed) == 80, "OctreeFileHeader.num_points_processed");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, records_offset) == 88, "OctreeFileHeader.records_offset");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, counters_offset) == 96, "OctreeFileHeader.counters_offset");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, samples_offset) == 104, "OctreeFileHeader.samples_offset");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, file_size) == 112, "OctreeFileHeader.file_size");
SIMLOD_STATIC_ASSERT(offsetof(SimlodOctreeFileHeader, reserved1) == 120, "OctreeFileHeader.reserved1");

// Region query and clip volumes (simlod_b200.h, DESIGN.md §9.8 and §9.15): kernel arguments of query.cu, render.cu and
// pick.cu
enum { SIMLOD_REGION_BOX = 1, SIMLOD_REGION_SPHERE = 2, SIMLOD_REGION_PLANES = 3 };
#define SIMLOD_REGION_MAX_PLANES 16
typedef struct SimlodRegion {
    uint32_t kind, num_planes;                      //   0  SIMLOD_REGION_*; planes in use (PLANES only)
    float    box_min[3], box_max[3];                //   8  BOX:    min <= p <= max on every axis
    float    center[3], radius;                     //  32  SPHERE: |p - center|^2 <= radius^2
    float    planes[SIMLOD_REGION_MAX_PLANES][4];   //  48  PLANES: n.p + d >= 0 for each of the first num_planes, (nx, ny, nz, d)
} SimlodRegion;
SIMLOD_STATIC_ASSERT(sizeof(SimlodRegion) == 304, "Region");
SIMLOD_STATIC_ASSERT(offsetof(SimlodRegion, box_min) == 8 && offsetof(SimlodRegion, box_max) == 20, "Region.box");
SIMLOD_STATIC_ASSERT(offsetof(SimlodRegion, center) == 32 && offsetof(SimlodRegion, radius) == 44, "Region.sphere");
SIMLOD_STATIC_ASSERT(offsetof(SimlodRegion, planes) == 48, "Region.planes");
enum { SIMLOD_CLIP_NONE = 0, SIMLOD_CLIP_INSIDE = 1, SIMLOD_CLIP_OUTSIDE = 2 };
#define SIMLOD_CLIP_MAX_REGIONS 4
typedef struct SimlodClip {
    uint32_t     mode, num_regions;                         //   0  SIMLOD_CLIP_*; regions in use
    SimlodRegion regions[SIMLOD_CLIP_MAX_REGIONS];          //   8  (304 bytes each)
} SimlodClip;
SIMLOD_STATIC_ASSERT(sizeof(SimlodClip) == 1224, "Clip");
SIMLOD_STATIC_ASSERT(offsetof(SimlodClip, regions) == 8, "Clip.regions");
