// nearest.cu — the k nearest samples of a batch of query positions (DESIGN.md §9.10), as indices into the export.
//
// Reads the ABI only, like the export (export.cu), whose plan, collect, scratch and chunk items it runs unchanged first.
// The candidates of a record are in its chunk items: with depth < 0 the points of a leaf, with depth >= 0 the points and
// voxels of a record of the cut. Every candidate lies in a record without children (a terminal record). Four kernels:
//
//   simlod_nearest_locate   one thread per query: a finite query descends the record tree by its lattice coordinate,
//                           clamped into the cube, to a terminal record, its home; a query with a non-finite coordinate
//                           gets the extra home numRecords (searched nowhere). Counts per home, a slot in its bucket.
//   simlod_nearest_scan     one block: exclusive scans of the counts (bucket offsets) and of the runs of up to
//                           NEAREST_RUN queries per home; checks that the record tree's levels step by one up to 20
//   simlod_nearest_scatter  one thread per query: its id into its home's bucket
//   simlod_nearest_search   one block per run. The block stages the home's candidates through shared memory once for its
//                           queries; each warp keeps its query's k best (d2, index) keys, one sorted slot per lane. Then
//                           each warp walks the record tree alone, depth first, children nearest first, skipping every
//                           record whose lattice box cannot hold a candidate that beats its k-th key, and writes its slots.
//
// Nothing is written outside the scratch and NearestCtl before the search, and the search writes only the destinations.
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
constexpr uint64_t NO_INDEX = ~0ull;                            // an empty slot: key (+inf, NO_INDEX) follows every sample
constexpr uint32_t INF_BITS = 0x7f800000u;

static_assert(RUN * 32 <= 1024 && SIMLOD_NEAREST_MAX_K <= 32, "one warp per query, one slot per lane");

// The key of a sample: (d2 bits, index). d2 is a sum of squares of finite differences, never NaN and never -0, so its
// bits order as the float does.
__device__ __forceinline__ bool keyLess(uint32_t d, uint64_t i, uint32_t kd, uint64_t ki) {
    return d < kd || (d == kd && i < ki);
}

// The warp's top-k: lane j < k holds slot j (d, index, source address), ascending. Every lane offers at most one
// candidate; those below the k-th key are inserted one at a time, lowest lane first (the result does not depend on the
// order: the key is a total order and no sample is offered twice).
struct TopK {
    uint32_t d = INF_BITS, kd = INF_BITS;
    uint64_t index = NO_INDEX, src = 0, kindex = NO_INDEX;

    __device__ __forceinline__ void offer(bool want, uint32_t cd, uint64_t ci, uint64_t cs, uint32_t lane, uint32_t k) {
        want = want && keyLess(cd, ci, kd, kindex);
        uint32_t m = __ballot_sync(FULL, want);
        while (m) {
            const uint32_t from = __ffs(m) - 1;
            const uint32_t nd = __shfl_sync(FULL, cd, from);
            const uint64_t ni = __shfl_sync(FULL, ci, from), ns = __shfl_sync(FULL, cs, from);
            const uint32_t pos = __popc(__ballot_sync(FULL, lane < k && keyLess(d, index, nd, ni)));   // < k
            const uint32_t ud = __shfl_up_sync(FULL, d, 1);
            const uint64_t ui = __shfl_up_sync(FULL, index, 1), us = __shfl_up_sync(FULL, src, 1);
            if (lane == pos) { d = nd; index = ni; src = ns; }
            else if (lane > pos) { d = ud; index = ui; src = us; }
            kd = __shfl_sync(FULL, d, k - 1);
            kindex = __shfl_sync(FULL, index, k - 1);
            want = want && lane != from && keyLess(cd, ci, kd, kindex);
            m = __ballot_sync(FULL, want);
        }
    }
};

// Grid-stride over the queries with whole warps (the bucket slots are taken one atomic per home and warp).
extern "C" __global__ void __launch_bounds__(256)
simlod_nearest_locate(const NearestArgs a) {
    const QueryCube c = queryCube(a.boxMin, a.boxMax);
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < a.numQueries; base += stride) {
        const uint32_t i = base + lane;
        uint32_t home = FULL;
        if (i < a.numQueries) {
            const float4 q = *(const float4*)(a.queries + 4ull * i);
            home = a.numRecords;
            if (isfinite(q.x) && isfinite(q.y) && isfinite(q.z)) {
                const float p[3] = {q.x, q.y, q.z}, mn[3] = {c.minx, c.miny, c.minz};
                uint32_t L[3];
#pragma unroll
                for (int ax = 0; ax < 3; ax++) {   // the lattice cell, clamped into the cube (fmax drops a NaN)
                    const double t = ((double)p[ax] - (double)mn[ax]) / (double)c.size * 1048576.0;
                    L[ax] = (uint32_t)fmin(fmax(t, 0.0), 1048575.0);
                }
                uint32_t r = 0;
                for (uint32_t level = 0; level < SIMLOD_MAX_DEPTH; level++) {
                    const int32_t fc = a.rec[r].first_child;
                    if (fc < 0) break;
                    const uint32_t sh = SIMLOD_MAX_DEPTH - 1 - level;
                    r = (uint32_t)fc + ((((L[0] >> sh) & 1u) << 2) | (((L[1] >> sh) & 1u) << 1) | ((L[2] >> sh) & 1u));
                }
                home = r;
            }
        }
        // one atomic per distinct home in the warp
        const uint32_t peers = __match_any_sync(FULL, home);
        const uint32_t leader = __ffs(peers) - 1;
        uint32_t first = 0;
        if (lane == leader && home != FULL) first = atomicAdd(&a.count[home], (uint32_t)__popc(peers));
        first = __shfl_sync(FULL, first, leader);
        if (home != FULL) {
            a.home[i] = home;
            a.slot[i] = first + __popc(peers & ((1u << lane) - 1u));
        }
    }
}

// One block: bucket offsets and run starts over the numRecords + 1 homes, and the record tree's levels: the root at 0,
// every child one below its parent, no inner record at level 20. With them the search's stack cannot overflow.
extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_nearest_scan(const NearestArgs a) {
    const uint32_t homes = a.numRecords + 1;
    uint64_t queryBase = 0, runBase = 0;
    bool bad = false;
    for (uint32_t tile = 0; tile < homes; tile += PLAN_THREADS) {
        const uint32_t r = tile + threadIdx.x;
        const uint32_t c = r < homes ? a.count[r] : 0;
        uint64_t tq = 0, tr = 0;
        const uint64_t pq = blockScan<false>(c, &tq);
        const uint64_t pr = blockScan<false>((c + RUN - 1) / RUN, &tr);
        if (r < homes) { a.offset[r] = (uint32_t)(queryBase + pq); a.runStart[r] = (uint32_t)(runBase + pr); }
        queryBase += tq; runBase += tr;
        if (r < a.numRecords && levelOutOfStep(a.rec, r)) bad = true;
    }
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) {
        a.runStart[homes] = (uint32_t)runBase;
        a.ctl->numRuns = (uint32_t)runBase;
        if (bad) a.ctl->error = EXPORT_ERR_CHILD;
    }
}

extern "C" __global__ void __launch_bounds__(256)
simlod_nearest_scatter(const NearestArgs a) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.numQueries; i += gridDim.x * blockDim.x)
        a.bucket[a.offset[a.home[i]] + a.slot[i]] = i;
}

// One warp offers the samples of chunk item `it` (global memory, 16-byte loads); points must be eligible.
__device__ __forceinline__ void offerItem(TopK& top, const uint64_t* __restrict__ items, uint64_t item, bool voxel, const QueryCube& c,
                                          float qx, float qy, float qz, float rr, uint32_t lane, uint32_t k) {
    const uint64_t src = items[2 * item], dst = items[2 * item + 1];
    const uint32_t n = (uint32_t)(dst >> 48);
    const uint64_t first = dst & 0xffffffffffffull;
    const uint4* __restrict__ s = (const uint4*)src;
    for (uint32_t j0 = 0; j0 < n; j0 += 32) {
        const uint32_t j = j0 + lane;
        bool want = false;
        uint32_t cd = INF_BITS;
        if (j < n) {
            const uint4 v = __ldg(s + j);
            const float x = __uint_as_float(v.x), y = __uint_as_float(v.y), z = __uint_as_float(v.z);
            const float d2 = dist2(x, y, z, qx, qy, qz);
            want = d2 <= rr && (voxel || inCube(c, x, y, z));
            cd = __float_as_uint(d2);
        }
        top.offer(want, cd, first + j, src + 16ull * j, lane, k);
    }
}

extern "C" __global__ void __launch_bounds__(RUN * 32)
simlod_nearest_search(const NearestArgs a) {
    __shared__ float4 shPos[TILE];                 // x, y, z of the staged candidates; x = NaN for an ineligible point
    __shared__ uint64_t shSrc[TILE];               // their addresses
    __shared__ uint32_t stRec[RUN][STACK];
    __shared__ double stBound[RUN][STACK];
    __shared__ unsigned long long shCount[4];      // found, tested, visited, invalid

    const uint32_t run = blockIdx.x;
    if (a.ctl->error || run >= a.ctl->numRuns) return;            // block-uniform
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, k = a.k;
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
    if (threadIdx.x < 4) shCount[threadIdx.x] = 0;
    __syncthreads();

    const QueryCube c = queryCube(a.boxMin, a.boxMax);
    const float4 q = active ? *(const float4*)(a.queries + 4ull * qid) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    const float rr = fpx::mul(a.maxRadius, a.maxRadius);
    TopK top;
    uint64_t tested = 0, visited = 0;
    const bool searched = home < a.numRecords;     // block-uniform: the other home holds the non-finite queries

    // the home's candidates, staged once for the block's queries
    if (searched) {
        const SimlodExportNode& h = a.rec[home];
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
                const uint64_t src = a.items[2 * item] + 16ull * (w % PPC);
                float4 p = __ldg((const float4*)src);
                if (!voxel && !inCube(c, p.x, p.y, p.z)) p.x = __int_as_float(0x7fffffff);
                shPos[j] = p;
                shSrc[j] = src;
            }
            __syncthreads();
            if (active) {
                for (uint32_t j0 = 0; j0 < n; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    bool want = false;
                    uint32_t cd = INF_BITS;
                    uint64_t src = 0;
                    if (j < n) {
                        const float4 p = shPos[j];
                        const float d2 = dist2(p.x, p.y, p.z, q.x, q.y, q.z);
                        want = d2 <= rr;                   // false for NaN: an ineligible point
                        cd = __float_as_uint(d2);
                        src = shSrc[j];
                    }
                    top.offer(want, cd, base + t0 + j, src, lane, k);
                }
            }
        }
        tested = count;
        visited = count ? 1 : 0;
    }

    // the rest of the tree, one warp per query, depth first from the root with the nearest child on top
    if (active && searched) {
        const double margin = searchMargin(c);
        uint32_t* const sRec = stRec[warp];
        double* const sBound = stBound[warp];
        if (lane == 0) { sRec[0] = 0; sBound[0] = 0.0; }
        uint32_t depthOfStack = 1;
        __syncwarp();
        while (depthOfStack > 0) {
            depthOfStack--;
            const uint32_t r = sRec[depthOfStack];
            const double bound = sBound[depthOfStack];
            __syncwarp();                          // read before a push overwrites it
            const double thr = skipAbove(top.kd, rr);
            if (bound > thr) continue;
            const SimlodExportNode& nd = a.rec[r];
            const int32_t fc = nd.first_child;
            if (fc < 0) {                          // terminal: its candidates, unless it is the home (done above)
                if (r == home) continue;
                const uint32_t np = nd.num_points;
                const uint64_t i0 = a.recItem[r];
                const uint32_t pointItems = ceilChunks(np);
                const uint32_t numItems = pointItems + (a.depth < 0 ? 0 : ceilChunks(nd.num_voxels));
                for (uint32_t it = 0; it < numItems; it++)
                    offerItem(top, a.items, i0 + it, it >= pointItems, c, q.x, q.y, q.z, rr, lane, k);
                tested += candidateCount(nd, a.depth);
                visited++;
                continue;
            }
            // inner: the children that may hold a better candidate, pushed farthest first
            const uint32_t child = (uint32_t)fc + (lane & 7u);
            bool keep = false;
            double cb = 0.0;
            if (lane < 8) {
                const SimlodExportNode& ch = a.rec[child];
                keep = ch.first_child >= 0 || candidateCount(ch, a.depth) > 0;
                if (keep) { cb = lowerBound(ch, c, margin, q.x, q.y, q.z); keep = !(cb > thr); }
            }
            const uint32_t kept = __ballot_sync(FULL, keep) & 0xffu;
            uint32_t pos = 0;                      // kept children after this one in (bound, child) descending order
#pragma unroll
            for (uint32_t o = 0; o < 8; o++) {
                const double ob = __shfl_sync(FULL, cb, o);
                if (((kept >> o) & 1u) && (ob > cb || (ob == cb && o > lane))) pos++;
            }
            if (keep) { sRec[depthOfStack + pos] = child; sBound[depthOfStack + pos] = cb; }
            depthOfStack += __popc(kept);
            __syncwarp();
        }
    }

    if (active) {
        if (lane < k) {
            const uint64_t o = (uint64_t)qid * k + lane;
            const bool filled = top.index != NO_INDEX;
            if (a.dstIndex) a.dstIndex[o] = filled ? (int64_t)top.index : -1;
            if (a.dstDist2) a.dstDist2[o] = __uint_as_float(top.d);
            if (a.dstSamples) ((uint4*)a.dstSamples)[o] = filled ? __ldg((const uint4*)top.src) : make_uint4(0, 0, 0, 0);
        }
        const uint32_t found = __popc(__ballot_sync(FULL, lane < k && top.index != NO_INDEX));
        if (lane == 0) {
            atomicAdd(&shCount[0], (unsigned long long)found);
            atomicAdd(&shCount[1], (unsigned long long)tested);
            atomicAdd(&shCount[2], (unsigned long long)visited);
            if (!searched) atomicAdd(&shCount[3], 1ull);
        }
    }
    __syncthreads();
    if (threadIdx.x < 4 && shCount[threadIdx.x]) {
        unsigned long long* const dst = (unsigned long long*)&a.ctl->numFound;
        atomicAdd(dst + threadIdx.x, shCount[threadIdx.x]);
    }
}
