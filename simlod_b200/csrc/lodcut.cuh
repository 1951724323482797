// lodcut.cuh — the renderer's per-node visibility and LOD-cut test (reference render.cu:762-933, math.cuh:55-64,154-201),
// shared by kernel_render (render.cu) and the view export (export.cu) so that both evaluate the same floating-point
// sequence. Every value that decides a flag is computed with the instruction sequence of the reference's SASS
// (fpmath.cuh, DESIGN.md §5).
#pragma once
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "fpmath.cuh"

// mat4 row * (x, y, z, 1): y*r.y -> fma(x, r.x) -> fma(z, r.z) -> + r.w   (helper_math.h:1266 as contracted in the reference SASS)
__device__ __forceinline__ float rowDot(const SimlodFloat4& r, float x, float y, float z) {
    return fpx::add(r.w, fpx::fma(z, r.z, fpx::fma(x, r.x, fpx::mul(y, r.y))));
}
// dot(float3, float3) with the same contraction
__device__ __forceinline__ float dot3(float ax, float ay, float az, float bx, float by, float bz) {
    return fpx::fma(az, bz, fpx::fma(ax, bx, fpx::mul(ay, by)));
}

// ------------------------------------------------------------------------------------------
// visibility, pass 1 (render.cu:762-901 + math.cuh:55-64,154-201)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ bool planeRejects(float px, float py, float pz, float pw,
                                             float minx, float miny, float minz, float maxx, float maxy, float maxz) {
    float len = fpx::sqrt_approx(dot3(px, py, pz, px, py, pz));        // length(): x*x + y*y + z*z, MUFU.SQRT
    float inv = fpx::rcp(len);
    float nx = fpx::mul_ftz(px, inv), ny = fpx::mul_ftz(py, inv), nz = fpx::mul_ftz(pz, inv);
    float constant = fpx::mul_ftz(pw, inv);
    float vx = nx > 0.0f ? maxx : minx;
    float vy = ny > 0.0f ? maxy : miny;
    float vz = nz > 0.0f ? maxz : minz;
    float d = fpx::add(dot3(nx, ny, nz, vx, vy, vz), constant);
    return d < 0.0f;
}

// edge of the octree's cube: the longest side of the box, as kernel_render derives it from the uniforms
__device__ __forceinline__ float cubeSizeOf(const SimlodUniforms& u) {
    float bsx = fpx::sub(u.boxMax[0], u.boxMin[0]);
    float bsy = fpx::sub(u.boxMax[1], u.boxMin[1]);
    float bsz = fpx::sub(u.boxMax[2], u.boxMin[2]);
    return fmaxf(fmaxf(bsx, bsy), bsz);
}

struct NodeBox { float mn[3], mx[3]; };
__device__ __forceinline__ NodeBox nodeBox(uint32_t level, uint32_t X, uint32_t Y, uint32_t Z, float cubeSize, float cminx, float cminy, float cminz) {
    NodeBox bx;
    float fx = fpx::u2f(X), fy = fpx::u2f(Y), fz = fpx::u2f(Z);
    float nodeSize = fpx::mul_ftz(cubeSize, fpx::ex2(-fpx::u2f(level)));      // cubeSize / pow(2, level)
    bx.mn[0] = fpx::fma(nodeSize, fx, cminx); bx.mn[1] = fpx::fma(nodeSize, fy, cminy); bx.mn[2] = fpx::fma(nodeSize, fz, cminz);
    bx.mx[0] = fpx::fma(nodeSize, fpx::add(fx, 1.0f), cminx); bx.mx[1] = fpx::fma(nodeSize, fpx::add(fy, 1.0f), cminy);
    bx.mx[2] = fpx::fma(nodeSize, fpx::add(fz, 1.0f), cminz);
    return bx;
}
// screen-space bounding rectangle of the 8 corners larger than 2 x minNodeSize in x or y (render.cu:783-818,880-890): a
// function of the node's coordinates alone
__device__ __forceinline__ bool boxIsLarge(const SimlodUniforms& u, const NodeBox& bx) {
    const SimlodFloat4* T = u.transform_updateBound.rows;
    float sminx = 0, smaxx = 0, sminy = 0, smaxy = 0;
#pragma unroll
    for (int corner = 0; corner < 8; corner++) {
        float x = (corner & 4) ? bx.mx[0] : bx.mn[0];
        float y = (corner & 2) ? bx.mx[1] : bx.mn[1];
        float z = (corner & 1) ? bx.mx[2] : bx.mn[2];
        float w = rowDot(T[3], x, y, z);
        float rw = fpx::rcp(w);
        float sx = fpx::mul(u.width, fpx::fma(fpx::mul_ftz(rowDot(T[0], x, y, z), rw), 0.5f, 0.5f));
        float sy = fpx::mul(u.height, fpx::fma(fpx::mul_ftz(rowDot(T[1], x, y, z), rw), 0.5f, 0.5f));
        if (corner == 0) { sminx = smaxx = sx; sminy = smaxy = sy; }
        else { sminx = fminf(sminx, sx); smaxx = fmaxf(smaxx, sx); sminy = fminf(sminy, sy); smaxy = fmaxf(smaxy, sy); }
    }
    float dx = fpx::sub(smaxx, sminx), dy = fpx::sub(smaxy, sminy);
    double limit = 2.0 * (double)u.minNodeSize;
    return (double)dx > limit || (double)dy > limit;
}
// frustum planes rows[3] -+ rows[0..2] (math.cuh:175-182)
__device__ __forceinline__ bool boxInFrustum(const SimlodUniforms& u, const NodeBox& bx) {
    const SimlodFloat4* T = u.transform_updateBound.rows;
    bool inFrustum = true;
#pragma unroll
    for (int p = 0; p < 6 && inFrustum; p++) {
        const SimlodFloat4& a = T[3];
        const SimlodFloat4& b = T[p == 0 || p == 1 ? 0 : (p == 2 || p == 3 ? 1 : 2)];
        bool minus = (p == 0 || p == 3 || p == 4);
        float px = minus ? fpx::sub(a.x, b.x) : fpx::add(a.x, b.x);
        float py = minus ? fpx::sub(a.y, b.y) : fpx::add(a.y, b.y);
        float pz = minus ? fpx::sub(a.z, b.z) : fpx::add(a.z, b.z);
        float pw = minus ? fpx::sub(a.w, b.w) : fpx::add(a.w, b.w);
        if (planeRejects(px, py, pz, pw, bx.mn[0], bx.mn[1], bx.mn[2], bx.mx[0], bx.mx[1], bx.mx[2])) inFrustum = false;
    }
    return inFrustum;
}

__device__ __forceinline__ bool isLeaf(const SimlodNode* node) {
    bool leaf = true;
#pragma unroll
    for (int i = 0; i < 8; i++) leaf = leaf && node->children[i] == nullptr;
    return leaf;
}

// One node's flags (render.cu:762-901) and whether the LOD cut draws it (render.cu:906-933): a visible non-large child
// of a large node, or a large visible leaf. The parent's `isLarge` is a function of the parent's coordinates
// (level - 1, X/2, Y/2, Z/2) and the frozen update transform alone, so it is recomputed here instead of read from the
// parent: the test needs no other node's flags and is evaluated for every node on its own. `visible` and `large` are
// the values kernel_render stores in Node::visible / Node::isLarge.
__device__ __forceinline__ bool nodeDrawn(const SimlodUniforms& u, const SimlodNode* node, float cubeSize,
                                          float cminx, float cminy, float cminz, bool& visible, bool& large) {
    const uint32_t level = node->level, X = node->X, Y = node->Y, Z = node->Z;
    const NodeBox bx = nodeBox(level, X, Y, Z, cubeSize, cminx, cminy, cminz);
    large = boxIsLarge(u, bx);
    const bool hasSamples = node->numPoints > 0 || node->numVoxels > 0;
    visible = hasSamples && boxInFrustum(u, bx);
    if (!visible) return false;
    if (large) return isLeaf(node);
    return level > 0 && boxIsLarge(u, nodeBox(level - 1, X >> 1, Y >> 1, Z >> 1, cubeSize, cminx, cminy, cminz));
}
