// splat.cuh — what kernel_render computes for one sample: its projection and the colour the frame displays (reference
// render.cu:49-78). Shared by kernel_render (render.cu) and the pick (pick.cu), so that a pick is decided by the frame's
// own floating-point sequence (fpmath.cuh, DESIGN.md §5).
#pragma once
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "fpmath.cuh"
#include "lodcut.cuh"

__constant__ uint32_t SPECTRAL[8] = {0x4f3ed5, 0x436df4, 0x61aefd, 0x8be0fe, 0x98f5e6, 0xa4ddab, 0xa5c266, 0xbd8832};

// Node::getID() % 127 (structures.cuh:116-143, render.cu:74-76) of a node or an export record (both carry the node's
// name), with its arithmetic as compiled: the first nine digits are shifted as 32-bit ints (wrap, then sign-extend into
// the 64-bit id), the rest as 64-bit values; unused name bytes are 0, i.e. digit -48. A template over the record type,
// so that the name is read through the record (whose alignment lets the loads be vectorised) and not a byte pointer.
template <class Record>
__device__ __forceinline__ uint32_t nodeColorId(const Record* node) {
    uint64_t id = node->name[0] == 'r' ? 1ull : 0ull;
#pragma unroll
    for (int k = 1; k <= 9; k++) {
        int32_t d = (int32_t)node->name[k] - 48;
        id |= (uint64_t)(int64_t)(int32_t)((uint32_t)d << (3 * k));
    }
    const int sh[9] = {30, 33, 36, 39, 42, 45, 48, 51, 53};
#pragma unroll
    for (int k = 10; k <= 18; k++) {
        int64_t d = (int64_t)((int32_t)node->name[k] - 48);
        id |= (uint64_t)d << sh[k - 10];
    }
    return (uint32_t)(id % 127ull);
}

// ------------------------------------------------------------------------------------------
// projection of one sample (render.cu:61-70)
// ------------------------------------------------------------------------------------------
struct Projected { int x, y; float depth; bool inside; };

__device__ __forceinline__ Projected project(const SimlodFloat4* T, float width, float height, float px, float py, float pz) {
    Projected r;
    float w = rowDot(T[3], px, py, pz);
    float rw = fpx::rcp(w);
    float ndcx = fpx::mul_ftz(rowDot(T[0], px, py, pz), rw);
    float ndcy = fpx::mul_ftz(rowDot(T[1], px, py, pz), rw);
    double dw = (double)width, dh = (double)height;
    r.x = fpx::d2i(fpx::dmul(fpx::dfma((double)ndcx, 0.5, 0.5), dw));       // int((ndc.x * 0.5 + 0.5) * width), in double
    r.y = fpx::d2i(fpx::dmul(fpx::dfma((double)ndcy, 0.5, 0.5), dh));
    r.depth = w;
    r.inside = r.x > 1 && (double)r.x < fpx::dadd(dw, -2.0) && r.y > 1 && (double)r.y < fpx::dadd(dh, -2.0);
    return r;
}

// the colour a sample is drawn with: its own, or by node (colorId = nodeColorId) or by level
__device__ __forceinline__ uint32_t sampleColor(const SimlodUniforms& u, uint32_t pointColor, uint32_t level, uint32_t colorId) {
    if (u.colorByNode) return (uint32_t)((uint64_t)colorId * 123456789ull);  // (node->getID() % 127) * 123456789 (render.cu:74-76)
    if (u.colorByLOD) {                                                      // render.cu:49-59,76-78
        int index = fpx::f2i(fpx::mul((float)(8 - (int)level), 1.8f));
        index = max(0, min(index, 7));
        return SPECTRAL[index];
    }
    return pointColor;
}
