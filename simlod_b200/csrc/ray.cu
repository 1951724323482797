// ray.cu — the first stored sample along each of a batch of rays (DESIGN.md §9.11), as an index into the export.
//
// Reads the ABI only, like the export (export.cu), whose plan, collect, scratch and chunk items it runs unchanged first.
// The samples of a record are in its chunk items: with depth < 0 the points of a leaf, with depth >= 0 the points and
// voxels of a record of the cut. Every sample lies in a record without children (a terminal record). Two kernels:
//
//   simlod_ray_check   one block: the record tree's levels step by one up to 20 (levelOutOfStep, which the k-nearest
//                      query's scan uses too), so that the trace's stack cannot overflow
//   simlod_ray_trace   one warp per ray, RAY_WARPS per block. The warp normalises the direction and walks the record
//                      tree alone, depth first from the root, the nearest child on top. Lanes 0-7 clip the ray against
//                      the 8 children's inflated lattice boxes; every lane tests a terminal record's samples, and a warp
//                      reduction of the (t, index) key updates the best hit, which shortens the clip of what follows.
//
// The trace returns at once when the check found the image inconsistent, so nothing is written into a destination
// unless the whole result is.
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "../../include/simlod_b200.h"
#include "lodcut.cuh"
#include "export_common.cuh"
#include "region.cuh"

constexpr uint32_t STACK = 7 * SIMLOD_MAX_DEPTH + 1;            // a pop adds at most 8, at most 20 levels deep
constexpr uint32_t FULL = 0xffffffffu;
constexpr uint64_t NO_INDEX = ~0ull;                            // no hit: key (+inf, NO_INDEX) follows every hit
constexpr uint64_t NO_KEY = ~0ull;                              // no hit in a record: above every (t bits, position)
constexpr uint32_t INF_BITS = 0x7f800000u;
constexpr uint32_t LOADS = 4;                                   // 16-byte sample loads in flight per lane

// A ray as the contract defines it (include/simlod_b200.h): its validity and its direction normalised in double, every
// operation .rn and uncontracted, so that numpy repeats it bit for bit.
struct Ray {
    float o[3], u[3], tmin, tmax;
    bool valid;
};

__device__ __forceinline__ Ray loadRay(const float* __restrict__ rays, uint32_t i) {
    const float4 a = *(const float4*)(rays + 8ull * i), b = *(const float4*)(rays + 8ull * i + 4);
    Ray r;
    r.o[0] = a.x; r.o[1] = a.y; r.o[2] = a.z; r.tmin = a.w; r.tmax = b.w;
    r.valid = isfinite(a.x) && isfinite(a.y) && isfinite(a.z) && isfinite(b.x) && isfinite(b.y) && isfinite(b.z) &&
              (b.x != 0.0f || b.y != 0.0f || b.z != 0.0f) && isfinite(a.w) && a.w >= 0.0f && b.w >= a.w;
    const double dx = fpx::f2d(b.x), dy = fpx::f2d(b.y), dz = fpx::f2d(b.z);
    const double len = fpx::dsqrt(fpx::dadd(fpx::dadd(fpx::dmul(dx, dx), fpx::dmul(dy, dy)), fpx::dmul(dz, dz)));
    r.u[0] = fpx::d2f(fpx::ddiv(dx, len)); r.u[1] = fpx::d2f(fpx::ddiv(dy, len)); r.u[2] = fpx::d2f(fpx::ddiv(dz, len));
    return r;
}

// t and h2 of a sample: w = p - o, t = ((wx*ux + wy*uy) + wz*uz) + 0 (no -0, so t's bits order as the float does),
// c = w x u, h2 = (cx*cx + cy*cy) + cz*cz, all float32 without contraction.
__device__ __forceinline__ void rayKey(const Ray& r, float x, float y, float z, float& t, float& h2) {
    const float wx = fpx::sub(x, r.o[0]), wy = fpx::sub(y, r.o[1]), wz = fpx::sub(z, r.o[2]);
    t = fpx::add(fpx::add(fpx::add(fpx::mul(wx, r.u[0]), fpx::mul(wy, r.u[1])), fpx::mul(wz, r.u[2])), 0.0f);
    const float cx = fpx::sub(fpx::mul(wy, r.u[2]), fpx::mul(wz, r.u[1]));
    const float cy = fpx::sub(fpx::mul(wz, r.u[0]), fpx::mul(wx, r.u[2]));
    const float cz = fpx::sub(fpx::mul(wx, r.u[1]), fpx::mul(wy, r.u[0]));
    h2 = fpx::add(fpx::add(fpx::mul(cx, cx), fpx::mul(cy, cy)), fpx::mul(cz, cz));
}

__device__ __forceinline__ uint32_t candidateCount(const SimlodExportNode& r, int32_t depth) {
    return depth < 0 ? r.num_points : r.num_points + r.num_voxels;
}

// The clip of a record (DESIGN.md §9.11): false when none of its samples can be a hit, else [lo, hi] with lo < t < hi
// for the float t of every sample of it that is a hit. `margin` bounds the eligible samples by the lattice box (§9.8);
// D bounds |p - o| in the 1-norm, and e = 2^-20 D covers the float error of t and of |c| (at most 7 and 6 units of
// 2^-24 D). `reach` bounds the distance of a hit from the line: radius (1 + 2^-20) + 1e-20, or +inf when r*r overflows.
// Evaluated in double; a NaN (a degenerate cube) clips nothing, and a zero component of u is never divided by.
__device__ __forceinline__ bool clip(const NodeBox& b, const double o[3], const double inv[3], const float u[3],
                                     double margin, double reach, double& lo, double& hi) {
    double D = 0.0;
#pragma unroll
    for (int a = 0; a < 3; a++)
        D += fmax(fabs(((double)b.mn[a] - margin) - o[a]), fabs(((double)b.mx[a] + margin) - o[a]));
    lo = -INFINITY; hi = INFINITY;
    if (!(D < 1e38)) return true;                  // products of such a sample may overflow: no bound
    const double e = D * 0x1p-20 + 1e-30;
    const double grow = margin + reach + e;
    double enter = -INFINITY, exit = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double l = ((double)b.mn[a] - grow) - o[a], h = ((double)b.mx[a] + grow) - o[a];
        if (u[a] == 0.0f) {                        // the ray never leaves its plane on this axis
            if (l > 0.0 || h < 0.0) return false;
        } else {
            const double s0 = l * inv[a], s1 = h * inv[a];
            enter = fmax(enter, fmin(s0, s1));
            exit = fmin(exit, fmax(s0, s1));
        }
    }
    lo = enter - e;
    hi = exit + e;
    return !(lo > hi);
}

// One block: the levels of the record tree (levelOutOfStep), so that the trace's stack of STACK entries cannot overflow
extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_ray_check(const RayArgs a) {
    bool bad = false;
    for (uint32_t r = threadIdx.x; r < a.numRecords; r += PLAN_THREADS)
        if (levelOutOfStep(a.rec, r)) bad = true;
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0 && bad) a.ctl->error = EXPORT_ERR_CHILD;
}

extern "C" __global__ void __launch_bounds__(RAY_WARPS * 32)
simlod_ray_trace(const RayArgs a) {
    __shared__ uint32_t stRec[RAY_WARPS][STACK];
    __shared__ double stLo[RAY_WARPS][STACK];
    __shared__ unsigned long long shCount[4];      // hits, tested, visited, invalid

    if (a.ctl->error) return;                      // block-uniform
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t id = blockIdx.x * RAY_WARPS + warp;
    if (threadIdx.x < 4) shCount[threadIdx.x] = 0;
    __syncthreads();

    if (id < a.numRays) {
        const Ray r = loadRay(a.rays, id);
        uint32_t bestT = INF_BITS, bestRec = 0, bestPos = 0;
        uint64_t bestIndex = NO_INDEX, tested = 0, visited = 0;
        if (r.valid && a.numRecords) {
            const QueryCube c = queryCube(a.boxMin, a.boxMax);
            const double cubeMax = fmax(fmax(fmax(fabs((double)c.minx), fabs((double)c.miny)), fabs((double)c.minz)),
                                        fmax(fmax(fabs((double)c.minx + c.size), fabs((double)c.miny + c.size)), fabs((double)c.minz + c.size)));
            const double margin = (double)c.size * 0x1p-19 + cubeMax * 0x1p-21;
            const float rr = fpx::mul(a.radius, a.radius);
            const double reach = isinf(rr) ? (double)INFINITY : (double)a.radius * (1.0 + 0x1p-20) + 1e-20;
            const double o[3] = {(double)r.o[0], (double)r.o[1], (double)r.o[2]};
            double inv[3];
#pragma unroll
            for (int ax = 0; ax < 3; ax++) inv[ax] = r.u[ax] != 0.0f ? 1.0 / (double)r.u[ax] : 0.0;
            uint32_t* const sRec = stRec[warp];
            double* const sLo = stLo[warp];
            if (lane == 0) { sRec[0] = 0; sLo[0] = -INFINITY; }
            uint32_t top = 1;
            __syncwarp();
            while (top > 0) {
                top--;
                const uint32_t rid = sRec[top];
                const double entry = sLo[top];
                __syncwarp();                      // read before a push overwrites it
                const double lim = fmin((double)__uint_as_float(bestT), (double)r.tmax);
                if (entry > lim) continue;         // every hit in it has t > lim: a later key, or beyond tmax
                const SimlodExportNode& nd = a.rec[rid];
                const int32_t fc = nd.first_child;
                if (fc < 0) {                      // terminal: every sample, the best (t bits, position) per lane
                    const uint32_t np = nd.num_points;
                    const uint64_t i0 = a.recItem[rid], base = nd.sample_offset;
                    const uint32_t pointItems = ceilChunks(np);
                    const uint32_t numItems = pointItems + (a.depth < 0 ? 0 : ceilChunks(nd.num_voxels));
                    uint64_t key = NO_KEY;
                    for (uint32_t it = 0; it < numItems; it++) {
                        const uint64_t src = a.items[2 * (i0 + it)], dst = a.items[2 * (i0 + it) + 1];
                        const uint32_t n = (uint32_t)(dst >> 48);
                        const uint32_t pos0 = (uint32_t)((dst & 0xffffffffffffull) - base);
                        const bool voxel = it >= pointItems;
                        const uint4* __restrict__ s = (const uint4*)src;
                        for (uint32_t j0 = 0; j0 < n; j0 += 32 * LOADS) {
                            uint4 v[LOADS];
#pragma unroll
                            for (uint32_t q = 0; q < LOADS; q++) {
                                const uint32_t j = j0 + 32 * q + lane;
                                if (j < n) v[q] = __ldg(s + j);
                            }
#pragma unroll
                            for (uint32_t q = 0; q < LOADS; q++) {
                                const uint32_t j = j0 + 32 * q + lane;
                                if (j < n) {
                                    const float x = __uint_as_float(v[q].x), y = __uint_as_float(v[q].y), z = __uint_as_float(v[q].z);
                                    float t, h2;
                                    rayKey(r, x, y, z, t, h2);
                                    if (t >= r.tmin && t <= r.tmax && h2 <= rr && (voxel || inCube(c, x, y, z)))
                                        key = min(key, (uint64_t)__float_as_uint(t) << 32 | (pos0 + j));
                                }
                            }
                        }
                    }
#pragma unroll
                    for (uint32_t off = 16; off; off >>= 1) key = min(key, (uint64_t)__shfl_xor_sync(FULL, key, off));
                    if (key != NO_KEY) {           // positions follow the indices, so this is the record's least (t, index)
                        const uint32_t kt = (uint32_t)(key >> 32), kp = (uint32_t)key;
                        if (kt < bestT || (kt == bestT && base + kp < bestIndex)) {
                            bestT = kt; bestIndex = base + kp; bestRec = rid; bestPos = kp;
                        }
                    }
                    tested += candidateCount(nd, a.depth);
                    visited++;
                    continue;
                }
                // inner: the children whose clip may hold a better hit, pushed farthest entry first
                const uint32_t child = (uint32_t)fc + (lane & 7u);
                bool keep = false;
                double clo = -INFINITY;
                if (lane < 8) {
                    const SimlodExportNode& ch = a.rec[child];
                    keep = ch.first_child >= 0 || candidateCount(ch, a.depth) > 0;
                    if (keep) {
                        const NodeBox b = nodeBox(ch.level, ch.X, ch.Y, ch.Z, c.size, c.minx, c.miny, c.minz);
                        double chi;
                        keep = clip(b, o, inv, r.u, margin, reach, clo, chi) && !(chi < (double)r.tmin) && !(clo > lim);
                        if (isnan(clo)) clo = -INFINITY;
                    }
                }
                const uint32_t kept = __ballot_sync(FULL, keep) & 0xffu;
                uint32_t pos = 0;                  // kept children after this one in (entry, child) descending order
#pragma unroll
                for (uint32_t k = 0; k < 8; k++) {
                    const double ok = __shfl_sync(FULL, clo, k);
                    if (((kept >> k) & 1u) && (ok > clo || (ok == clo && k > lane))) pos++;
                }
                if (keep) { sRec[top + pos] = child; sLo[top + pos] = clo; }
                top += __popc(kept);
                __syncwarp();
            }
        }
        if (lane == 0) {
            const bool hit = bestIndex != NO_INDEX;
            float h2 = __uint_as_float(INF_BITS);
            uint4 sample = make_uint4(0, 0, 0, 0);
            if (hit) {                             // the sample again, for its bytes and its h2
                const SimlodExportNode& br = a.rec[bestRec];
                const uint32_t np = br.num_points;
                const bool voxel = bestPos >= np;
                const uint32_t w = voxel ? bestPos - np : bestPos;
                const uint64_t item = a.recItem[bestRec] + (voxel ? ceilChunks(np) : 0) + w / PPC;
                sample = __ldg((const uint4*)a.items[2 * item] + w % PPC);
                float t;
                rayKey(r, __uint_as_float(sample.x), __uint_as_float(sample.y), __uint_as_float(sample.z), t, h2);
            }
            if (a.dstIndex) a.dstIndex[id] = hit ? (int64_t)bestIndex : -1;
            if (a.dstT) a.dstT[id] = __uint_as_float(bestT);
            if (a.dstH2) a.dstH2[id] = h2;
            if (a.dstSamples) ((uint4*)a.dstSamples)[id] = sample;
            if (hit) atomicAdd(&shCount[0], 1ull);
            if (tested) atomicAdd(&shCount[1], (unsigned long long)tested);
            if (visited) atomicAdd(&shCount[2], (unsigned long long)visited);
            if (!r.valid) atomicAdd(&shCount[3], 1ull);
        }
    }
    __syncthreads();
    if (threadIdx.x < 4 && shCount[threadIdx.x]) {
        unsigned long long* const dst = (unsigned long long*)&a.ctl->numHits;
        atomicAdd(dst + threadIdx.x, shCount[threadIdx.x]);
    }
}
