// export_common.cuh — what the export (export.cu) and the region query (query.cu) share: the control word, the chunk
// item, the inconsistency codes and the block-wide scan of their one-block plan kernels.
#pragma once
#include <stdint.h>
#include "../../include/simlod_abi.h"

constexpr uint32_t PLAN_THREADS = 1024;
constexpr uint32_t PPC = SIMLOD_POINTS_PER_CHUNK;

enum : uint32_t {                         // ExportCtl::error (the canonicaliser's codes, oracle.cpp canonFromImage)
    EXPORT_ERR_CHILD = 1,                 // a child pointer outside nodes[] (or more records than nodes: a node reached twice)
    EXPORT_ERR_CHUNK = 2,                 // a chunk pointer outside the used heap
    EXPORT_ERR_SHORT = 4,                 // a list shorter than its count
    EXPORT_ERR_PARTIAL = 5,               // an inner node without all 8 children
};

struct ExportCtl {                        // mirrors host.cpp
    uint32_t numNodes, maxLevel;
    uint64_t numSamples, numPoints, numVoxels;
    uint64_t numItems;
    uint32_t error, pad;
};

struct Item { uint64_t src; uint64_t dst; };   // dst: sample index | count << 48

__device__ __forceinline__ uint32_t ceilChunks(uint32_t n) { return (n + PPC - 1) / PPC; }

// Block-wide exclusive scan (PLAN_THREADS threads) of 64-bit values; returns the prefix, *total the sum. One instance per
// plan kernel (isView), so that each kernel has its own warpSums and the full / depth plan keeps its shared-memory layout.
template <bool isView>
__device__ uint64_t blockScan(uint64_t v, uint64_t* total) {
    __shared__ uint64_t warpSums[PLAN_THREADS / 32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint64_t x = v;
    for (uint32_t o = 1; o < 32; o <<= 1) {
        uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warpSums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint64_t s = warpSums[lane];
        for (uint32_t o = 1; o < 32; o <<= 1) {
            uint64_t y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        warpSums[lane] = s;
    }
    __syncthreads();
    const uint64_t prefix = (warp ? warpSums[warp - 1] : 0) + x - v;
    *total = warpSums[PLAN_THREADS / 32 - 1];
    __syncthreads();                       // warpSums is reused by the next call
    return prefix;
}
