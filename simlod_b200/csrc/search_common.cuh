// search_common.cuh — what the searches by distance (nearest.cu, radius.cu) share: the float32 squared distance of their
// key, the candidates of a terminal record, and the lower bound and threshold by which a record is skipped unread
// (DESIGN.md §9.10).
#pragma once
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "lodcut.cuh"
#include "region.cuh"

__device__ __forceinline__ float dist2(float x, float y, float z, float qx, float qy, float qz) {
    const float dx = fpx::sub(x, qx), dy = fpx::sub(y, qy), dz = fpx::sub(z, qz);
    return fpx::add(fpx::add(fpx::mul(dx, dx), fpx::mul(dy, dy)), fpx::mul(dz, dz));
}

// The candidates of a terminal record, and its chunk items: points first, then (depth >= 0) voxels
__device__ __forceinline__ uint32_t candidateCount(const SimlodExportNode& r, int32_t depth) {
    return depth < 0 ? r.num_points : r.num_points + r.num_voxels;
}

// The inflation of a lattice box that holds every eligible sample of its record (§9.8): 2 cells + 2^-21 of the largest
// coordinate magnitude of the cube
__device__ __forceinline__ double searchMargin(const QueryCube& c) {
    const double cubeMax = fmax(fmax(fmax(fabs((double)c.minx), fabs((double)c.miny)), fabs((double)c.minz)),
                                fmax(fmax(fabs((double)c.minx + c.size), fabs((double)c.miny + c.size)), fabs((double)c.minz + c.size)));
    return (double)c.size * 0x1p-19 + cubeMax * 0x1p-21;
}

// Lower bound of the exact squared distance from q to any eligible sample of a record, by §9.8's argument (query.cu
// regionMisses): the lattice box inflated by `margin`, evaluated in double. fmax drops a NaN, so the bound is never NaN.
__device__ __forceinline__ double lowerBound(const SimlodExportNode& r, const QueryCube& c, double margin, float qx, float qy, float qz) {
    const NodeBox b = nodeBox(r.level, r.X, r.Y, r.Z, c.size, c.minx, c.miny, c.minz);
    const float q[3] = {qx, qy, qz};
    double d2 = 0.0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double lo = (double)b.mn[a] - margin, hi = (double)b.mx[a] + margin, v = (double)q[a];
        const double d = fmax(fmax(lo - v, v - hi), 0.0);
        d2 += d * d;
    }
    return d2;
}

// A record is skipped when its bound exceeds this: the float key of a sample beyond it is above min(k-th key, r*r),
// since the float sum's relative error is below 2^-21 (twice that allowed) and 1e-44 covers products that underflow.
// Strictly above: such a sample cannot tie the k-th key either. +inf (fewer than k found, no radius) skips nothing.
__device__ __forceinline__ double skipAbove(uint32_t kd, float rr) {
    return (double)fminf(__uint_as_float(kd), rr) * (1.0 + 0x1p-20) + 1e-44;
}
