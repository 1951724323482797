// region.cuh — the two per-sample predicates of the region query (DESIGN.md §9.8), stated once for the count and the
// write kernel of query.cu, and the clip test that render.cu and pick.cu build on the first of them (§9.15). Every operation is an explicit fpx:: instruction (round to nearest, no contraction), so the
// numpy float32 restatement of the tests (tests/query_restatement.py) agrees in the last bit.
#pragma once
#include <stdint.h>
#include "../../include/simlod_b200.h"
#include "fpmath.cuh"

// The octree cube as the builder derives it from the uniforms (construct.cu, voxels.cu:860-863)
struct QueryCube { float minx, miny, minz, size, rcpSize; };

__device__ __forceinline__ QueryCube queryCube(const float* boxMin, const float* boxMax) {
    QueryCube c;
    c.minx = boxMin[0]; c.miny = boxMin[1]; c.minz = boxMin[2];
    c.size = fmaxf(fmaxf(fpx::sub(boxMax[0], boxMin[0]), fpx::sub(boxMax[1], boxMin[1])), fpx::sub(boxMax[2], boxMin[2]));
    c.rcpSize = fpx::rcp(c.size);
    return c;
}

// Point predicate: whether (x, y, z) lies in the region.
__device__ __forceinline__ bool regionContains(const SimlodRegion& r, float x, float y, float z) {
    if (r.kind == SIMLOD_REGION_BOX)
        return x >= r.box_min[0] && x <= r.box_max[0] && y >= r.box_min[1] && y <= r.box_max[1] && z >= r.box_min[2] && z <= r.box_max[2];
    if (r.kind == SIMLOD_REGION_SPHERE) {
        const float dx = fpx::sub(x, r.center[0]), dy = fpx::sub(y, r.center[1]), dz = fpx::sub(z, r.center[2]);
        return fpx::add(fpx::add(fpx::mul(dx, dx), fpx::mul(dy, dy)), fpx::mul(dz, dz)) <= fpx::mul(r.radius, r.radius);
    }
    bool in = true;
    for (uint32_t k = 0; k < r.num_planes; k++) {
        const float v = fpx::add(fpx::add(fpx::add(fpx::mul(r.planes[k][0], x), fpx::mul(r.planes[k][1], y)), fpx::mul(r.planes[k][2], z)), r.planes[k][3]);
        in = in && v >= 0.0f;
    }
    return in;
}

// Clip predicate of render.cu and pick.cu (DESIGN.md §9.15): whether a sample at (x, y, z) is drawn under `c`. It is in
// when regionContains holds for one of the first num_regions regions; INSIDE keeps what is in, OUTSIDE what is not, NONE
// everything.
__device__ __forceinline__ bool clipKeeps(const SimlodClip& c, float x, float y, float z) {
    if (c.mode == SIMLOD_CLIP_NONE) return true;
    bool in = false;
    for (uint32_t k = 0; k < c.num_regions && !in; k++) in = regionContains(c.regions[k], x, y, z);
    return c.mode == SIMLOD_CLIP_OUTSIDE ? !in : in;
}

// In-cube predicate: the point is not below boxMin and its 2^20 lattice coordinate (the builder's quantize(), construct.cu)
// is below 2^20 on every axis. Only for such a point is the coordinate the builder descended by the point's own, so only
// such a point is bounded by the box of the node that stores it.
__device__ __forceinline__ bool inCubeAxis(float p, float mn, float rcpSize) {
    return p >= mn && fpx::f2u(fpx::mul_ftz(fpx::mul(fpx::add(p, -mn), 1048576.0f), rcpSize)) < 1048576u;
}
__device__ __forceinline__ bool inCube(const QueryCube& c, float x, float y, float z) {
    return inCubeAxis(x, c.minx, c.rcpSize) && inCubeAxis(y, c.miny, c.rcpSize) && inCubeAxis(z, c.minz, c.rcpSize);
}
