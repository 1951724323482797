// export_common.cuh — what the export (export.cu) and the queries built on its plan (query.cu, pick.cu, nearest.cu, ray.cu)
// share: the chunk item, the block-wide scan of the one-block plan kernels and the record tree's level check. The control
// word and its inconsistency codes are in kernel_args.h.
#pragma once
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "kernel_args.h"

constexpr uint32_t PLAN_THREADS = 1024;
constexpr uint32_t PPC = SIMLOD_POINTS_PER_CHUNK;

struct Item { uint64_t src; uint64_t dst; };   // dst: sample index | count << 48

__device__ __forceinline__ uint32_t ceilChunks(uint32_t n) { return (n + PPC - 1) / PPC; }

// The record that chunk item k belongs to: the last one whose first item is <= k (recItem is non-decreasing; records
// without items share a value with the next record)
__device__ __forceinline__ uint32_t itemRecord(uint64_t k, const uint64_t* __restrict__ recItem, uint32_t n) {
    uint32_t lo = 0, hi = n;               // recItem[lo] <= k < recItem[hi] (recItem[n] = numItems)
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (recItem[mid] <= k) lo = mid; else hi = mid;
    }
    return lo;
}

// Whether record r breaks the level rule the searches of nearest.cu and ray.cu rely on: the root at level 0, every
// child one level below its parent, no inner record at level 20. With it a depth-first walk that pushes at most 8 children
// per pop never holds more than 7 * 20 + 1 records.
__device__ __forceinline__ bool levelOutOfStep(const SimlodExportNode* rec, uint32_t r) {
    const SimlodExportNode& n = rec[r];
    bool bad = r == 0 && n.level != 0;
    if (n.first_child >= 0) {
        if (n.level >= SIMLOD_MAX_DEPTH) bad = true;
        for (uint32_t k = 0; k < 8; k++) bad = bad || rec[(uint32_t)n.first_child + k].level != n.level + 1;
    }
    return bad;
}

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
