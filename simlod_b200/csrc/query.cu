// query.cu — region query: the samples of the octree inside a box, a sphere or a convex set of half-spaces, filtered
// into a flat array in a deterministic order (DESIGN.md §9.8).
//
// Reads the ABI only, like the export (export.cu), whose scratch, control word, chunk items and collect kernel it shares.
// Four kernels of its own, with simlod_export_collect between the first two:
//
//   simlod_query_plan    one block: breadth-first from the root as simlod_export_plan, except that every node is first
//                        classified against the region from its lattice box. A node that cannot hold a passing sample is
//                        OUTSIDE: its children and lists are not read and it is not expanded. The records of the other
//                        (visited) nodes carry the counts of the lists the sample set takes from them.
//   simlod_export_collect  (export.cu) one item per chunk of those lists, every pointer tested before it is dereferenced
//   simlod_query_count   warps take items (<= 1000 samples): 16-byte loads, both predicates, ballot + popc; one count per item
//   simlod_query_scan    one block: exclusive scan of the item counts into destination offsets, totals into QueryCtl
//   simlod_query_write   after the host has checked QueryCtl: items are read and tested again and the passing samples
//                        stored in slot order at the item's offset, so the destination order is the source order
//
// Nothing is written outside the scratch, QueryCtl and, in the last kernel, the destination.
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "../../include/simlod_b200.h"
#include "lodcut.cuh"
#include "export_common.cuh"
#include "region.cuh"

constexpr uint64_t VOXEL_ITEM = 1ull << 63;   // item word: count (after the scan: destination offset) | VOXEL_ITEM

// Whether no eligible sample stored in a node with box `b` can pass the point predicate of `r`. Conservative: `false` is
// always allowed. The box is inflated by `margin` on every side first. A stored eligible point has the lattice
// coordinate X the builder descended by, X / 2^(20 - level) is the node's coordinate, and
//   * X = trunc(fl(fl(dx * 2^20) * rcp)) with rcp = MUFU.RCP(size) (relative error < 2^-21 together with the rounding of
//     the product) puts dx / size * 2^20 within (X - 0.5, X + 1.5) since X < 2^20; dx = fl(p - min) adds 2^-4 cell;
//   * nodeBox() computes the node's corners with a relative error < 2^-21 of the cube edge (MUFU.EX2, one product: half a
//     cell) and one fma rounding (half an ulp of the corner, at most 2^-24 of the largest coordinate of the cube),
// so the point lies within 1.1 cells + 2^-24 maxAbs of the computed box. margin = 2 cells + 2^-21 maxAbs leaves the rest
// for the roundings of the test itself, which is evaluated in double. The float predicates round as well: the sphere's
// sum has a relative error < 2^-21 and a plane's an absolute error < 2^-22 (|nx x| + |ny y| + |nz z| + |d|); both tests
// allow twice that, plus 1e-44 for products that underflow. Comparisons are written so that a NaN means "not outside".
__device__ __forceinline__ bool regionMisses(const SimlodRegion& r, const NodeBox& b, double margin) {
    double mn[3], mx[3];
#pragma unroll
    for (int a = 0; a < 3; a++) { mn[a] = (double)b.mn[a] - margin; mx[a] = (double)b.mx[a] + margin; }
    if (r.kind == SIMLOD_REGION_BOX) {
        bool out = false;
#pragma unroll
        for (int a = 0; a < 3; a++) out = out || (double)r.box_max[a] < mn[a] || (double)r.box_min[a] > mx[a];
        return out;
    }
    if (r.kind == SIMLOD_REGION_SPHERE) {
        double d2 = 0.0;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const double c = (double)r.center[a];
            const double d = fmax(fmax(mn[a] - c, c - mx[a]), 0.0);       // distance to the nearest point of the box
            d2 += d * d;
        }
        const double rr = (double)r.radius * (double)r.radius;
        return d2 > rr * (1.0 + 0x1p-20) + 1e-44;
    }
    bool out = false;
    for (uint32_t k = 0; k < r.num_planes; k++) {
        double v = (double)r.planes[k][3], mag = fabs(v);
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const double n = (double)r.planes[k][a];
            v += n * (n > 0.0 ? mx[a] : mn[a]);                            // the p-vertex: the corner furthest along n
            mag += fabs(n) * fmax(fabs(mn[a]), fabs(mx[a]));
        }
        out = out || v < -(mag * 0x1p-21 + 1e-44);
    }
    return out;
}

// depth < 0: the points of every leaf. depth >= 0: the export's cut at `depth`. Scratch as simlod_export_plan; of a
// record only num_points, num_voxels and sample_offset are written (what simlod_export_collect reads).
extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_query_plan(const uint8_t* __restrict__ nodes, const SimlodStats* __restrict__ stats, int32_t depth, uint32_t maxRecords,
                  SimlodExportNode* __restrict__ rec, uint32_t* __restrict__ recNode, uint64_t* __restrict__ recItem,
                  QueryCtl* __restrict__ ctl, const SimlodRegion region, const QueryBox box) {
    __shared__ uint32_t sh_total, sh_error, sh_maxLevel, sh_visited;
    const uint32_t numNodes = stats->numNodes;
    const uint64_t nodesAddr = (uint64_t)nodes;
    if (threadIdx.x == 0) {
        sh_total = 1; sh_error = 0; sh_maxLevel = 0; sh_visited = 0;
        if (numNodes == 0 || numNodes > maxRecords) sh_error = EXPORT_ERR_CHILD;
        recNode[0] = 0;
    }
    __syncthreads();
    if (sh_error) { if (threadIdx.x == 0) ctl->plan.error = sh_error; return; }

    const QueryCube cube = queryCube(box.mn, box.mx);
    const double maxAbs = fmax(fmax(fmax(fabs((double)cube.minx), fabs((double)cube.miny)), fabs((double)cube.minz)),
                               fmax(fmax(fabs((double)cube.minx + cube.size), fabs((double)cube.miny + cube.size)), fabs((double)cube.minz + cube.size)));
    const double margin = (double)cube.size * 0x1p-19 + maxAbs * 0x1p-21;

    // deepest level in the octree: every allocated node
    uint32_t lmax = 0;
    for (uint32_t i = threadIdx.x; i < numNodes; i += PLAN_THREADS)
        lmax = max(lmax, ((const SimlodNode*)(nodes + (uint64_t)i * sizeof(SimlodNode)))->level);
    atomicMax(&sh_maxLevel, lmax);

    uint32_t begin = 0, end = 1;
    for (int32_t level = 0; begin < end; level++) {
        const bool expand = depth < 0 || level < depth;
        for (uint32_t tile = begin; tile < end; tile += PLAN_THREADS) {
            const uint32_t r = tile + threadIdx.x;
            const bool valid = r < end;
            uint32_t numChildren = 0, err = 0;
            uint64_t child[8];
            const SimlodNode* node = nullptr;
            bool visited = false;
            if (valid) {
                node = (const SimlodNode*)(nodes + (uint64_t)recNode[r] * sizeof(SimlodNode));
                visited = !regionMisses(region, nodeBox(node->level, node->X, node->Y, node->Z, cube.size, cube.minx, cube.miny, cube.minz), margin);
            }
            if (visited) {
                #pragma unroll
                for (int k = 0; k < 8; k++) {
                    child[k] = (uint64_t)node->children[k];
                    if (child[k]) {
                        numChildren++;
                        const uint64_t off = child[k] - nodesAddr;
                        if (child[k] < nodesAddr || off % sizeof(SimlodNode) != 0 || off / sizeof(SimlodNode) >= numNodes) err = EXPORT_ERR_CHILD;
                    }
                }
                if (numChildren != 0 && numChildren != 8) err = EXPORT_ERR_PARTIAL;
            }
            const bool inner = numChildren == 8;
            uint64_t total = 0;
            const uint32_t pos = (uint32_t)blockScan<false>(visited && expand && inner && !err ? 8 : 0, &total);
            const uint32_t first = sh_total + pos;
            __syncthreads();
            if (threadIdx.x == 0) {
                if (sh_total + total > numNodes) atomicMax(&sh_error, EXPORT_ERR_CHILD);   // more records than nodes
                else sh_total += (uint32_t)total;
            }
            if (err) atomicMax(&sh_error, err);
            if (valid) {
                if (visited && expand && inner && !err && first + 8 <= numNodes) {
                    #pragma unroll
                    for (int k = 0; k < 8; k++) recNode[first + k] = (uint32_t)((child[k] - nodesAddr) / sizeof(SimlodNode));
                }
                const bool takePoints = visited && !inner, takeVoxels = visited && inner && level == depth;
                rec[r].num_points = takePoints ? node->numPoints : 0;
                rec[r].num_voxels = takeVoxels ? node->numVoxelsStored : 0;
                if (takePoints || takeVoxels) atomicAdd(&sh_visited, 1u);
            }
            __syncthreads();
            if (sh_error) break;
        }
        if (sh_error) break;
        begin = end;
        end = sh_total;
    }
    __syncthreads();
    if (sh_error) { if (threadIdx.x == 0) ctl->plan.error = sh_error; return; }

    // candidate sample offsets and chunk items: exclusive scans over the records
    const uint32_t n = sh_total;
    uint64_t samplesBase = 0, itemsBase = 0, points = 0, voxels = 0;
    for (uint32_t tile = 0; tile < n; tile += PLAN_THREADS) {
        const uint32_t r = tile + threadIdx.x;
        uint32_t np = 0, nv = 0;
        if (r < n) { np = rec[r].num_points; nv = rec[r].num_voxels; }
        uint64_t tS = 0, tI = 0, tP = 0, tV = 0;
        const uint64_t s = blockScan<false>((uint64_t)np + nv, &tS);
        const uint64_t it = blockScan<false>(ceilChunks(np) + ceilChunks(nv), &tI);
        blockScan<false>(np, &tP);
        blockScan<false>(nv, &tV);
        if (r < n) { rec[r].sample_offset = samplesBase + s; recItem[r] = itemsBase + it; }
        samplesBase += tS; itemsBase += tI; points += tP; voxels += tV;
    }
    if (threadIdx.x == 0) {
        ctl->plan.numNodes = n; ctl->plan.maxLevel = sh_maxLevel;
        ctl->plan.numSamples = samplesBase; ctl->plan.numPoints = points; ctl->plan.numVoxels = voxels;
        ctl->plan.numItems = itemsBase; ctl->plan.error = 0;
        ctl->outSamples = ctl->outPoints = ctl->outVoxels = 0;
        ctl->nodesVisited = sh_visited;
    }
}

constexpr uint32_t FILTER_UNROLL = 4;

// One warp filters the `count` samples at `src`: a sample passes when it lies in the region and, for a point, in the
// cube. Returns the number that pass; with `write`, stores them at dst in slot order. The count pass reads through the
// cache hierarchy, so that the write pass of a small region finds the samples in L2; the write pass streams.
template <bool write>
__device__ __forceinline__ uint32_t filterItem(const uint4* __restrict__ src, uint32_t count, bool voxel, const SimlodRegion& region,
                                               const QueryCube& cube, uint32_t lane, uint4* __restrict__ dst) {
    uint32_t passed = 0;
    for (uint32_t b = 0; b < count; b += 32 * FILTER_UNROLL) {
        uint4 v[FILTER_UNROLL];
        #pragma unroll
        for (uint32_t u = 0; u < FILTER_UNROLL; u++) {
            const uint32_t j = b + u * 32 + lane;
            if (j < count) v[u] = write ? __ldcs(src + j) : __ldcg(src + j);
        }
        #pragma unroll
        for (uint32_t u = 0; u < FILTER_UNROLL; u++) {
            const uint32_t j = b + u * 32 + lane;
            bool pass = false;
            if (j < count) {
                const float x = __uint_as_float(v[u].x), y = __uint_as_float(v[u].y), z = __uint_as_float(v[u].z);
                pass = regionContains(region, x, y, z) && (voxel || inCube(cube, x, y, z));
            }
            const uint32_t ballot = __ballot_sync(0xffffffffu, pass);
            if (write && pass) __stcs(dst + passed + __popc(ballot & ((1u << lane) - 1u)), v[u]);
            passed += __popc(ballot);
        }
    }
    return passed;
}

// Whether item k holds voxels: the items of a record are those of its point list, then those of its voxel list.
__device__ __forceinline__ bool itemIsVoxel(uint64_t k, const SimlodExportNode* __restrict__ rec, const uint64_t* __restrict__ recItem, uint32_t n) {
    const uint32_t r = itemRecord(k, recItem, n);
    return k - recItem[r] >= ceilChunks(rec[r].num_points);
}

extern "C" __global__ void __launch_bounds__(256)
simlod_query_count(const Item* __restrict__ items, const SimlodExportNode* __restrict__ rec, const uint64_t* __restrict__ recItem,
                   uint64_t* __restrict__ itemWord, const QueryCtl* __restrict__ ctl, const SimlodRegion region, const QueryBox box) {
    if (ctl->plan.error) return;           // the items are complete only when the plan and the collect found no error
    const QueryCube cube = queryCube(box.mn, box.mx);
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t numWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t numItems = ctl->plan.numItems;
    const uint32_t n = ctl->plan.numNodes;
    for (uint64_t k = warp; k < numItems; k += numWarps) {
        const Item it = items[k];
        const bool voxel = itemIsVoxel(k, rec, recItem, n);
        const uint32_t passed = filterItem<false>((const uint4*)it.src, (uint32_t)(it.dst >> 48), voxel, region, cube, lane, nullptr);
        if (lane == 0) itemWord[k] = passed | (voxel ? VOXEL_ITEM : 0);
    }
}

constexpr uint32_t SCAN_ITEMS = 8;         // consecutive items per thread and tile

// One block: itemWord[k] = the number of returned samples before item k (VOXEL_ITEM kept), and the totals.
extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_query_scan(uint64_t* __restrict__ itemWord, QueryCtl* __restrict__ ctl) {
    if (ctl->plan.error) return;
    const uint64_t numItems = ctl->plan.numItems;
    uint64_t base = 0, voxels = 0;
    for (uint64_t tile = 0; tile < numItems; tile += PLAN_THREADS * SCAN_ITEMS) {
        const uint64_t k0 = tile + (uint64_t)threadIdx.x * SCAN_ITEMS;
        uint64_t w[SCAN_ITEMS], sum = 0;
        #pragma unroll
        for (uint32_t i = 0; i < SCAN_ITEMS; i++) {
            w[i] = k0 + i < numItems ? itemWord[k0 + i] : 0;
            sum += w[i] & ~VOXEL_ITEM;
            if (w[i] & VOXEL_ITEM) voxels += w[i] & ~VOXEL_ITEM;
        }
        uint64_t total = 0;
        uint64_t at = base + blockScan<false>(sum, &total);
        #pragma unroll
        for (uint32_t i = 0; i < SCAN_ITEMS; i++) {
            if (k0 + i < numItems) itemWord[k0 + i] = at | (w[i] & VOXEL_ITEM);
            at += w[i] & ~VOXEL_ITEM;
        }
        base += total;
    }
    uint64_t voxelTotal = 0;
    blockScan<false>(voxels, &voxelTotal);
    if (threadIdx.x == 0) { ctl->outSamples = base; ctl->outVoxels = voxelTotal; ctl->outPoints = base - voxelTotal; }
}

extern "C" __global__ void __launch_bounds__(256)
simlod_query_write(const Item* __restrict__ items, const uint64_t* __restrict__ itemWord, uint4* __restrict__ dstSamples,
                   const QueryCtl* __restrict__ ctl, const SimlodRegion region, const QueryBox box) {
    const QueryCube cube = queryCube(box.mn, box.mx);
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t numWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t numItems = ctl->plan.numItems;
    for (uint64_t k = warp; k < numItems; k += numWarps) {
        const Item it = items[k];
        const uint64_t w = itemWord[k];
        const uint64_t next = k + 1 < numItems ? itemWord[k + 1] & ~VOXEL_ITEM : ctl->outSamples;
        if (next == (w & ~VOXEL_ITEM)) continue;           // nothing of this item passed: not read again
        filterItem<true>((const uint4*)it.src, (uint32_t)(it.dst >> 48), (w & VOXEL_ITEM) != 0, region, cube, lane, dstSamples + (w & ~VOXEL_ITEM));
    }
}
