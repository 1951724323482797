// Prints size and offset of every field of the host/device records, and the constants the kernels are built with,
// one "Record.field offset size" line each. Built against include/simlod_abi.h (ours), or with -DSIMLOD_ABI_REFERENCE
// against the reference's OWN headers (modules/progressive_octree); tests/test_abi_and_library.py requires the two
// listings to be identical, the reference's being stored in tests/golden/reference.json.
//   HostDeviceInterface.h  Uniforms, Stats, mat4     (host <-> device interface of the three kernels)
//   structures.cuh         Point, Chunk, OccupancyGrid, Node and the constants the kernels are built with
#include <cstddef>
#include <cstdint>
#include <cstdio>
#ifdef SIMLOD_ABI_REFERENCE
#include "HostDeviceInterface.h"      // reference
#include "helper_math.h"              // reference: dot() used by structures.cuh
#include "structures.cuh"             // reference
typedef Point P; typedef Chunk Ch; typedef OccupancyGrid G; typedef Node N; typedef Uniforms U; typedef Stats S; typedef mat4 M;
static const unsigned long long CONSTANTS[] = {MAX_POINTS_PER_NODE, POINTS_PER_CHUNK, MAX_DEPTH, GRID_NUM_CELLS / 32u, BATCH_STREAM_SIZE};
#else
#include "simlod_abi.h"               // ours
typedef SimlodPoint P; typedef SimlodChunk Ch; typedef SimlodOccupancyGrid G; typedef SimlodNode N; typedef SimlodUniforms U;
typedef SimlodStats S; typedef SimlodMat4 M;
static const unsigned long long CONSTANTS[] = {SIMLOD_MAX_POINTS_PER_NODE, SIMLOD_POINTS_PER_CHUNK, SIMLOD_MAX_DEPTH, SIMLOD_GRID_WORDS,
                                               SIMLOD_BATCH_STREAM_SIZE};
#endif

#define FIELD(T, f) std::printf("%s.%s %zu %zu\n", #T, #f, offsetof(T, f), sizeof(((T*)nullptr)->f))

int main() {
    std::printf("sizes %zu %zu %zu %zu %zu %zu %zu\n", sizeof(P), sizeof(Ch), sizeof(N), sizeof(G), sizeof(U), sizeof(S), sizeof(M));
    std::printf("constants %llu %llu %llu %llu %llu\n", CONSTANTS[0], CONSTANTS[1], CONSTANTS[2], CONSTANTS[3], CONSTANTS[4]);
    FIELD(P, x); FIELD(P, y); FIELD(P, z); FIELD(P, color);
    FIELD(Ch, points); FIELD(Ch, size); FIELD(Ch, next);
    FIELD(G, values);

    FIELD(N, children); FIELD(N, counter); FIELD(N, numPoints);
    FIELD(N, level); FIELD(N, X); FIELD(N, Y); FIELD(N, Z);
    FIELD(N, countIteration); FIELD(N, countFlag); FIELD(N, name);
    FIELD(N, visible); FIELD(N, isFiltered); FIELD(N, isLeaf); FIELD(N, isLarge);
    FIELD(N, grid); FIELD(N, points); FIELD(N, voxelChunks);
    FIELD(N, numVoxels); FIELD(N, numVoxelsStored);

    FIELD(U, width); FIELD(U, height); FIELD(U, time);
    FIELD(U, fovy_rad); FIELD(U, world); FIELD(U, view);
    FIELD(U, proj); FIELD(U, transform); FIELD(U, transform_updateBound);
    FIELD(U, transformInv_updateBound); FIELD(U, persistentBufferCapacity);
    FIELD(U, momentaryBufferCapacity); FIELD(U, frameCounter);
    FIELD(U, boxMin); FIELD(U, boxMax);
    FIELD(U, showBoundingBox); FIELD(U, showPoints); FIELD(U, colorByNode);
    FIELD(U, colorByLOD); FIELD(U, colorWhite); FIELD(U, doUpdateVisibility);
    FIELD(U, doProgressive); FIELD(U, LOD); FIELD(U, useHighQualityShading);
    FIELD(U, minNodeSize); FIELD(U, pointSize); FIELD(U, updateStats);
    FIELD(U, enableEDL); FIELD(U, edlStrength);

    FIELD(S, frameID); FIELD(S, numNodes); FIELD(S, numInner); FIELD(S, numLeaves);
    FIELD(S, numNonemptyLeaves); FIELD(S, numPoints); FIELD(S, numVoxels);
    FIELD(S, allocatedBytes_momentary); FIELD(S, allocatedBytes_persistent);
    FIELD(S, numVisibleNodes); FIELD(S, numVisibleInner); FIELD(S, numVisibleLeaves);
    FIELD(S, numVisiblePoints); FIELD(S, numVisibleVoxels); FIELD(S, numChunksPoints);
    FIELD(S, numChunksVoxels); FIELD(S, batchletIndex); FIELD(S, numPointsProcessed);
    FIELD(S, numAllocatedChunks); FIELD(S, chunkPoolSize); FIELD(S, dbg);
    FIELD(S, memCapacityReached);
    return 0;
}
