// radius.cu — every sample within a radius of each of a batch of query positions (DESIGN.md §9.12), as CSR indices into
// the export.
//
// Reads the ABI only, like the export (export.cu), whose plan, collect, scratch and chunk items it runs unchanged first,
// and then nearest.cu's simlod_nearest_locate / scan / scatter, which bucket the queries by their home record and check
// the record tree's levels. Every candidate lies in a record without children (a terminal record). Four kernels:
//
//   simlod_radius_count    one block per run of up to NEAREST_RUN queries with one home, one warp per query. The block
//                          stages the home's candidates through shared memory once for its queries; each warp then walks
//                          the rest of the record tree alone, depth first in octant order, skipping every record whose
//                          lattice box cannot hold a neighbour. Writes the query's total and its neighbours in terminal
//                          records before the home in Z-order, and sums the counts into RadiusCtl.
//   simlod_radius_reduce   one block per tile of RADIUS_SCAN_TILE totals: the tile's sum
//   simlod_radius_scan     the same tiles: the sum of the tiles before (from the reduce), then the exclusive scan of the
//                          tile's totals into offsets; the last tile writes offsets[numQueries]
//   simlod_radius_write    the count's grid and walk: each record's neighbours at a running cursor, positions within a
//                          round of 32 by ballot prefix, and the staged home's at offsets[q] + before[q]
//
// Terminal records come in Z-order: a depth-first walk that takes the children in octant order visits them so, and the
// home, staged first, is placed by its Z-key. So the result does not depend on how queries are bucketed or scheduled.
// Every kernel returns at once when the nearest scan found the image inconsistent; the host launches the write only
// after it has read the counts, so nothing is written into a destination unless the whole result is.
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "../../include/simlod_b200.h"
#include "lodcut.cuh"
#include "export_common.cuh"
#include "region.cuh"
#include "search_common.cuh"

constexpr uint32_t RUN = NEAREST_RUN;
constexpr uint32_t TILE = 1024;                                 // home candidates staged in shared memory per round
constexpr uint32_t STACK = 7 * SIMLOD_MAX_DEPTH + 1;            // a pop adds at most 8, at most 20 levels deep
constexpr uint32_t FULL = 0xffffffffu;
constexpr uint32_t INF_BITS = 0x7f800000u;

static_assert(RUN * 32 <= 1024, "one warp per query");

// The Z-order key of a record: morton(X, Y, Z at its level) << 3 * (20 - level), the child index bits x<<2 | y<<1 | z
// per level, root first. Distinct for distinct terminal records (their cells are disjoint).
__device__ __forceinline__ uint64_t spread3(uint32_t v) {
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

__device__ __forceinline__ uint64_t zKey(const SimlodExportNode& r) {
    return ((spread3(r.X) << 2) | (spread3(r.Y) << 1) | spread3(r.Z)) << (3 * (SIMLOD_MAX_DEPTH - r.level));
}

// One warp writes the neighbours among a round of up to 32 candidates: lane j's at cursor + (neighbours of the lanes
// below it). Returns the round's neighbours.
__device__ __forceinline__ uint32_t writeRound(const RadiusArgs& a, bool hit, uint64_t cursor, uint64_t index, float d2,
                                               uint4 sample, uint32_t lane) {
    const uint32_t m = __ballot_sync(FULL, hit);
    if (hit) {
        const uint64_t o = cursor + __popc(m & ((1u << lane) - 1u));
        if (a.dstIndex) a.dstIndex[o] = (int64_t)index;
        if (a.dstDist2) a.dstDist2[o] = d2;
        if (a.dstSamples) ((uint4*)a.dstSamples)[o] = sample;
    }
    return __popc(m);
}

// The count pass (WRITE false) and the write pass (WRITE true): the same runs, staging and walk.
template <bool WRITE>
__device__ __forceinline__ void radiusPass(const RadiusArgs& a) {
    __shared__ float4 shPos[TILE];                 // the staged candidates, bit for bit; x = NaN for an ineligible point
    __shared__ uint32_t stRec[RUN][STACK];
    __shared__ unsigned long long shCount[4];      // found, tested, visited, invalid
    __shared__ uint32_t shMax;

    const uint32_t run = blockIdx.x;
    if (a.nearestCtl->error || run >= a.nearestCtl->numRuns) return;      // block-uniform
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t homes = a.numRecords + 1;
    uint32_t lo = 0, hi = homes;                   // the home of this run: runStart[lo] <= run < runStart[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a.runStart[mid] <= run) lo = mid; else hi = mid;
    }
    const uint32_t home = lo;
    const uint32_t firstInHome = (run - a.runStart[home]) * RUN;
    const uint32_t numQ = min(RUN, a.count[home] - firstInHome);
    const bool active = warp < numQ;
    const uint32_t qid = active ? a.bucket[a.offset[home] + firstInHome + warp] : 0;
    if (!WRITE) {
        if (threadIdx.x < 4) shCount[threadIdx.x] = 0;
        if (threadIdx.x == 0) shMax = 0;
    }
    __syncthreads();

    const QueryCube c = queryCube(a.boxMin, a.boxMax);
    const float4 q = active ? *(const float4*)(a.queries + 4ull * qid) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    const float rr = fpx::mul(a.radius, a.radius);
    const bool searched = home < a.numRecords;     // block-uniform: the other home holds the non-finite queries
    uint64_t homeHits = 0, cursor = 0;             // write pass: the home's neighbours go to offsets[q] + before[q]
    if (WRITE && active) cursor = (uint64_t)a.offsets[qid] + a.before[qid];
    uint64_t tested = 0, visited = 0;

    // the home's candidates, staged once for the block's queries
    uint64_t homeKey = 0;
    if (searched) {
        const SimlodExportNode& h = a.rec[home];
        homeKey = zKey(h);
        const uint32_t np = h.num_points, count = candidateCount(h, a.depth);
        const uint64_t firstItem = a.recItem[home], base = h.sample_offset;
        for (uint32_t t0 = 0; t0 < count; t0 += TILE) {
            const uint32_t n = min(TILE, count - t0);
            __syncthreads();                       // the previous tile has been read
            for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
                const uint32_t s = t0 + j;
                const bool voxel = s >= np;
                const uint32_t w = voxel ? s - np : s;
                const uint64_t item = firstItem + (voxel ? ceilChunks(np) : 0) + w / PPC;
                float4 p = __ldg((const float4*)(a.items[2 * item] + 16ull * (w % PPC)));
                if (!voxel && !inCube(c, p.x, p.y, p.z)) p.x = __int_as_float(0x7fffffff);
                shPos[j] = p;
            }
            __syncthreads();
            if (active) {
                for (uint32_t j0 = 0; j0 < n; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    bool hit = false;
                    float d2 = 0.0f;
                    float4 p = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                    if (j < n) {
                        p = shPos[j];
                        d2 = dist2(p.x, p.y, p.z, q.x, q.y, q.z);
                        hit = d2 <= rr;                    // false for NaN: an ineligible point
                    }
                    if (WRITE) {
                        const uint4 bits = make_uint4(__float_as_uint(p.x), __float_as_uint(p.y), __float_as_uint(p.z), __float_as_uint(p.w));
                        homeHits += writeRound(a, hit, cursor + homeHits, base + t0 + j, d2, bits, lane);
                    } else {
                        homeHits += __popc(__ballot_sync(FULL, hit));
                    }
                }
            }
        }
        tested = count;
        visited = count ? 1 : 0;
    }

    // the rest of the tree, one warp per query, depth first from the root in octant order (Z-order)
    uint64_t found = homeHits, before = 0;
    if (WRITE && active) cursor = (uint64_t)a.offsets[qid];
    if (active && searched) {
        const double margin = searchMargin(c);
        const double thr = skipAbove(INF_BITS, rr);            // §9.10's threshold with the k-th key at +inf
        bool passed = false;                       // write pass: the walk has passed the home's place in Z-order
        uint32_t* const sRec = stRec[warp];
        if (lane == 0) sRec[0] = 0;
        uint32_t depthOfStack = 1;
        __syncwarp();
        while (depthOfStack > 0) {
            depthOfStack--;
            const uint32_t r = sRec[depthOfStack];
            __syncwarp();                          // read before a push overwrites it
            const SimlodExportNode& nd = a.rec[r];
            const int32_t fc = nd.first_child;
            if (fc < 0) {                          // terminal: its candidates, unless it is the home (done above)
                if (r == home) continue;
                const bool early = zKey(nd) < homeKey;
                if (WRITE && !early && !passed) { cursor += homeHits; passed = true; }
                const uint32_t np = nd.num_points;
                const uint64_t i0 = a.recItem[r];
                const uint32_t pointItems = ceilChunks(np);
                const uint32_t numItems = pointItems + (a.depth < 0 ? 0 : ceilChunks(nd.num_voxels));
                uint64_t hits = 0;
                for (uint32_t it = 0; it < numItems; it++) {
                    const bool voxel = it >= pointItems;
                    const uint64_t src = a.items[2 * (i0 + it)], dst = a.items[2 * (i0 + it) + 1];
                    const uint32_t n = (uint32_t)(dst >> 48);
                    const uint64_t first = dst & 0xffffffffffffull;
                    const uint4* __restrict__ s = (const uint4*)src;
                    for (uint32_t j0 = 0; j0 < n; j0 += 32) {
                        const uint32_t j = j0 + lane;
                        bool hit = false;
                        float d2 = 0.0f;
                        uint4 v = make_uint4(0, 0, 0, 0);
                        if (j < n) {
                            v = __ldg(s + j);
                            const float x = __uint_as_float(v.x), y = __uint_as_float(v.y), z = __uint_as_float(v.z);
                            d2 = dist2(x, y, z, q.x, q.y, q.z);
                            hit = d2 <= rr && (voxel || inCube(c, x, y, z));
                        }
                        if (WRITE) hits += writeRound(a, hit, cursor + hits, first + j, d2, v, lane);
                        else hits += __popc(__ballot_sync(FULL, hit));
                    }
                }
                if (WRITE) cursor += hits;
                found += hits;
                if (early) before += hits;
                tested += candidateCount(nd, a.depth);
                visited++;
                continue;
            }
            // inner: the children whose box may hold a neighbour, pushed so that octant 0 is popped first
            const uint32_t child = (uint32_t)fc + (lane & 7u);
            bool keep = false;
            if (lane < 8) {
                const SimlodExportNode& ch = a.rec[child];
                keep = ch.first_child >= 0 || candidateCount(ch, a.depth) > 0;
                if (keep) keep = !(lowerBound(ch, c, margin, q.x, q.y, q.z) > thr);
            }
            const uint32_t kept = __ballot_sync(FULL, keep) & 0xffu;
            if (keep) sRec[depthOfStack + __popc(kept >> (lane + 1))] = child;
            depthOfStack += __popc(kept);
            __syncwarp();
        }
    }

    if (!WRITE) {
        if (active && lane == 0) {
            a.total[qid] = (uint32_t)found;
            a.before[qid] = (uint32_t)before;
            atomicAdd(&shCount[0], (unsigned long long)found);
            atomicAdd(&shCount[1], (unsigned long long)tested);
            atomicAdd(&shCount[2], (unsigned long long)visited);
            if (!searched) atomicAdd(&shCount[3], 1ull);
            atomicMax(&shMax, (uint32_t)found);
        }
        __syncthreads();
        if (threadIdx.x < 4 && shCount[threadIdx.x]) {
            unsigned long long* const dst = (unsigned long long*)&a.ctl->numFound;
            atomicAdd(dst + threadIdx.x, shCount[threadIdx.x]);
        }
        if (threadIdx.x == 0 && shMax) atomicMax(&a.ctl->maxFound, shMax);
    }
}

extern "C" __global__ void __launch_bounds__(RUN * 32)
simlod_radius_count(const RadiusArgs a) {
    radiusPass<false>(a);
}

extern "C" __global__ void __launch_bounds__(RUN * 32)
simlod_radius_write(const RadiusArgs a) {
    radiusPass<true>(a);
}

// The totals of scan tile blockIdx.x, RADIUS_SCAN_ITEMS consecutive ones per thread
__device__ __forceinline__ uint64_t tileTotals(const RadiusArgs& a, uint32_t v[RADIUS_SCAN_ITEMS]) {
    const uint64_t first = (uint64_t)blockIdx.x * RADIUS_SCAN_TILE + (uint64_t)threadIdx.x * RADIUS_SCAN_ITEMS;
    uint64_t s = 0;
#pragma unroll
    for (uint32_t i = 0; i < RADIUS_SCAN_ITEMS; i++) {
        v[i] = first + i < a.numQueries ? a.total[first + i] : 0;
        s += v[i];
    }
    return s;
}

extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_radius_reduce(const RadiusArgs a) {
    if (a.nearestCtl->error) return;
    uint32_t v[RADIUS_SCAN_ITEMS];
    uint64_t sum = 0;
    blockScan<false>(tileTotals(a, v), &sum);
    if (threadIdx.x == 0) a.tileSum[blockIdx.x] = sum;
}

extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_radius_scan(const RadiusArgs a) {
    if (a.nearestCtl->error) return;
    uint64_t before = 0, tileBase = 0, tileSum = 0;
    for (uint32_t t = threadIdx.x; t < blockIdx.x; t += PLAN_THREADS) before += a.tileSum[t];
    blockScan<false>(before, &tileBase);           // the sum of the tiles before this one
    uint32_t v[RADIUS_SCAN_ITEMS];
    uint64_t o = tileBase + blockScan<false>(tileTotals(a, v), &tileSum);
    const uint64_t first = (uint64_t)blockIdx.x * RADIUS_SCAN_TILE + (uint64_t)threadIdx.x * RADIUS_SCAN_ITEMS;
#pragma unroll
    for (uint32_t i = 0; i < RADIUS_SCAN_ITEMS; i++) {
        if (first + i < a.numQueries) a.offsets[first + i] = (int64_t)o;
        o += v[i];
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) a.offsets[a.numQueries] = (int64_t)(tileBase + tileSum);
}
