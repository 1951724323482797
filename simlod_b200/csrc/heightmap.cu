// heightmap.cu — height maps (DESIGN.md §9.14): per cell of an x-y grid, the count, lowest, highest and mean z of the
// stored samples that fall in it, and the highest sample itself, as an index into the export.
//
// Reads the ABI only, like the export (export.cu), whose plan, collect, scratch and chunk items it runs unchanged first.
// The per-cell accumulators live in the context's query scratch and are reset by memsets (not launches). Two kernels:
//
//   simlod_heightmap_accumulate  warps take chunk items, gridded like simlod_query_count. An item whose record's
//                                inflated lattice box cannot hold a sample of a cell of the grid is skipped after one read
//                                of its record (gridMisses). Otherwise each sample is read once with a 16-byte streaming
//                                load and binned; lanes whose samples share a cell find each other with __match_any_sync,
//                                reduce within that group, and the group's leader issues one atomic per kept field.
//   simlod_heightmap_finalize    one thread per cell turns the accumulators into the destinations; the top sample's bytes
//                                come from its chunk item, found by binary search. Non-empty cells are summed per block.
//
// The count accumulator is always kept (the info's num_binned and nonempty_cells come from it); the minimum, the top key
// and the fixed-point sum only when a destination needs them. Nothing is written outside the scratch and the destinations.
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "../../include/simlod_b200.h"
#include "lodcut.cuh"
#include "export_common.cuh"
#include "region.cuh"

constexpr uint32_t FULL = 0xffffffffu;
constexpr uint32_t NO_CELL = 0xffffffffu;       // a lane without a binned sample (cells < 2^27)
constexpr uint32_t LOADS = 4;                   // 16-byte sample loads in flight per lane
constexpr uint32_t NAN_BITS = 0x7fc00000u;      // the z of an empty cell

// The sign-aware bit order of a float: -0 below +0, every negative below every positive
__device__ __forceinline__ uint32_t ordered(float z) {
    const uint32_t b = __float_as_uint(z);
    return b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float unordered(uint32_t o) {
    return __uint_as_float(o ^ ((o >> 31) ? 0x80000000u : 0xffffffffu));
}

// The grid's x (or y) range in double: no sample outside [lo, hi] can fall in a cell of the grid. A binned sample has
// u = fl(fl(x - ox) / cell) with u >= 0 and u < nx:
//   * x < ox gives fl(x - ox) < 0 (a non-zero difference of two floats never rounds to 0), so u >= 0 holds only for
//     u = -0, i.e. |fl(x - ox)| / cell < 2^-149, and then x > ox - cell 2^-148 (|x - ox| <= |fl(x - ox)| (1 + 2^-23));
//   * u < nx with nx exact in float and rounding monotonic gives fl(x - ox) / cell < nx, so x - ox < nx cell (1 + 2^-23).
// lo and hi widen both by far more than that and by 2^-50 |ox| for their own double roundings.
struct GridRange { double lo, hi; };
__device__ __forceinline__ GridRange gridRange(float o, float cell, uint32_t n) {
    const double od = (double)o, c = (double)cell, slack = fabs(od) * 0x1p-50;
    return GridRange{od - c * 0x1p-140 - slack, od + (double)n * c * (1.0 + 0x1p-20) + slack};
}

// Whether no eligible sample stored in a record with box `b` can fall in a cell of the grid. Conservative: an eligible
// sample of the record lies within `margin` of the computed lattice box (regionMisses in query.cu states why, for the
// same margin of 2 cells + 2^-21 maxAbs, with the rest of it left for the roundings of a double test like this one),
// and no sample outside the ranges of gridRange() is binned. A NaN compares false and keeps the record.
__device__ __forceinline__ bool gridMisses(const NodeBox& b, double margin, const GridRange& gx, const GridRange& gy) {
    return (double)b.mx[0] + margin < gx.lo || (double)b.mn[0] - margin > gx.hi ||
           (double)b.mx[1] + margin < gy.lo || (double)b.mn[1] - margin > gy.hi;
}

// (256, 1): without the minimum ptxas holds the kernel at 64 registers and spills 8 bytes; it needs 77, 3 blocks per SM
extern "C" __global__ void __launch_bounds__(256, 1)
simlod_heightmap_accumulate(const HeightmapArgs a) {
    __shared__ unsigned long long shCount[3];      // binned, tested, visited
    if (threadIdx.x < 3) shCount[threadIdx.x] = 0;
    __syncthreads();

    const QueryCube c = queryCube(a.boxMin, a.boxMax);
    const double maxAbs = fmax(fmax(fmax(fabs((double)c.minx), fabs((double)c.miny)), fabs((double)c.minz)),
                               fmax(fmax(fabs((double)c.minx + c.size), fabs((double)c.miny + c.size)), fabs((double)c.minz + c.size)));
    const double margin = (double)c.size * 0x1p-19 + maxAbs * 0x1p-21;
    const GridRange gx = gridRange(a.origin[0], a.cell, a.nx), gy = gridRange(a.origin[1], a.cell, a.ny);
    const double minz = fpx::f2d(c.minz);
    const double K = fpx::ddiv(0x1p30, fpx::f2d(c.size));
    const bool wantMin = a.zmin != nullptr, wantTop = a.top != nullptr, wantSum = a.sum != nullptr;

    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t numWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    uint64_t binned = 0, tested = 0, visited = 0;
    for (uint64_t k = warp; k < a.numItems; k += numWarps) {
        const uint32_t r = itemRecord(k, a.recItem, a.numRecords);
        const SimlodExportNode& nd = a.rec[r];
        const uint64_t first = a.recItem[r];
        const bool voxel = k - first >= ceilChunks(nd.num_points);
        if (a.depth < 0 && (voxel || nd.first_child >= 0)) continue;     // depth < 0: the points of the leaves only
        if (gridMisses(nodeBox(nd.level, nd.X, nd.Y, nd.Z, c.size, c.minx, c.miny, c.minz), margin, gx, gy)) continue;
        const uint64_t src = a.items[2 * k], dst = a.items[2 * k + 1];
        const uint32_t n = (uint32_t)(dst >> 48);
        const uint32_t index0 = (uint32_t)(dst & 0xffffffffffffull);   // < 2^32: the host refuses larger exports
        if (lane == 0) { tested += n; visited += k == first; }
        const uint4* __restrict__ s = (const uint4*)src;
        for (uint32_t j0 = 0; j0 < n; j0 += 32 * LOADS) {
            uint4 v[LOADS];
#pragma unroll
            for (uint32_t q = 0; q < LOADS; q++) {
                const uint32_t j = j0 + 32 * q + lane;
                if (j < n) v[q] = __ldcs(s + j);
            }
#pragma unroll
            for (uint32_t q = 0; q < LOADS; q++) {
                const uint32_t j = j0 + 32 * q + lane;
                uint32_t id = NO_CELL;
                float z = 0.0f;
                if (j < n) {
                    const float x = __uint_as_float(v[q].x), y = __uint_as_float(v[q].y);
                    z = __uint_as_float(v[q].z);
                    const float u = fpx::div_rn(fpx::sub(x, a.origin[0]), a.cell);
                    const float w = fpx::div_rn(fpx::sub(y, a.origin[1]), a.cell);
                    if (u >= 0.0f && w >= 0.0f && (voxel || inCube(c, x, y, z))) {     // a NaN fails before f2u
                        const uint32_t i = fpx::f2u(u), jj = fpx::f2u(w);
                        if (i < a.nx && jj < a.ny) id = jj * a.nx + i;
                    }
                }
                const uint32_t peers = __match_any_sync(FULL, id);
                if (id == NO_CELL) continue;       // the whole group: the reductions below name only its lanes
                binned++;
                const bool leader = lane == (uint32_t)__ffs(peers) - 1;
                const uint32_t oz = ordered(z);
                if (leader) atomicAdd(a.count + id, (uint32_t)__popc(peers));
                if (wantMin) {
                    const uint32_t m = __reduce_min_sync(peers, oz);
                    if (leader) atomicMin(a.zmin + id, m);
                }
                if (wantTop) {                     // the highest z, then among equal z the smallest index
                    const uint32_t hi = __reduce_max_sync(peers, oz);
                    const uint32_t lo = __reduce_max_sync(peers, oz == hi ? 0xffffffffu - (index0 + j) : 0u);
                    if (leader) atomicMax(a.top + id, (unsigned long long)hi << 32 | lo);
                }
                if (wantSum) {                     // q = rint(((double)z - minz) K); the group's sum exact mod 2^64
                    const uint64_t qw = (uint64_t)__double2ll_rn(fpx::dmul(fpx::dadd(fpx::f2d(z), -minz), K));
                    const uint32_t s0 = __reduce_add_sync(peers, (uint32_t)(qw & 0x1fffffu));
                    const uint32_t s1 = __reduce_add_sync(peers, (uint32_t)((qw >> 21) & 0x1fffffu));
                    const uint32_t s2 = __reduce_add_sync(peers, (uint32_t)(qw >> 42));
                    if (leader) atomicAdd(a.sum + id, (unsigned long long)s0 + ((unsigned long long)s1 << 21) + ((unsigned long long)s2 << 42));
                }
            }
        }
    }
    if (binned) atomicAdd(&shCount[0], (unsigned long long)binned);
    if (tested) atomicAdd(&shCount[1], (unsigned long long)tested);
    if (visited) atomicAdd(&shCount[2], (unsigned long long)visited);
    __syncthreads();
    if (threadIdx.x < 3 && shCount[threadIdx.x]) atomicAdd((unsigned long long*)&a.ctl->numBinned + threadIdx.x, shCount[threadIdx.x]);
}

// The 16 bytes of sample `index` of the export: its chunk item is the last whose first index is <= index (the items'
// first indices increase with the item number, and every item holds at least one sample)
__device__ __forceinline__ uint4 exportSample(const uint64_t* __restrict__ items, uint64_t numItems, uint64_t index) {
    uint64_t lo = 0, hi = numItems;                // first(lo) <= index < first(hi), first(numItems) = +inf
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) >> 1;
        if ((items[2 * mid + 1] & 0xffffffffffffull) <= index) lo = mid; else hi = mid;
    }
    const uint64_t first = items[2 * lo + 1] & 0xffffffffffffull;
    return __ldg((const uint4*)items[2 * lo] + (index - first));
}

extern "C" __global__ void __launch_bounds__(256)
simlod_heightmap_finalize(const HeightmapArgs a) {
    __shared__ unsigned long long shNonempty;
    if (threadIdx.x == 0) shNonempty = 0;
    __syncthreads();
    const QueryCube c = queryCube(a.boxMin, a.boxMax);
    const double minz = fpx::f2d(c.minz);
    const double K = fpx::ddiv(0x1p30, fpx::f2d(c.size));
    const float nan = __uint_as_float(NAN_BITS);
    const uint64_t cells = (uint64_t)a.nx * a.ny;
    uint32_t nonempty = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t n = a.count[i];
        nonempty += n != 0;
        if (a.dstCount) a.dstCount[i] = n;
        if (a.dstZMin) a.dstZMin[i] = n ? unordered(a.zmin[i]) : nan;
        if (a.dstZMean) {
            float mean = nan;
            if (n) {
                const double S = __ll2double_rn((long long)a.sum[i]);
                mean = fpx::d2f(fpx::dadd(minz, fpx::ddiv(fpx::ddiv(S, (double)n), K)));
            }
            a.dstZMean[i] = mean;
        }
        if (a.top) {
            const uint64_t key = n ? a.top[i] : 0;
            const uint64_t index = 0xffffffffull - (uint32_t)key;
            if (a.dstZMax) a.dstZMax[i] = n ? unordered((uint32_t)(key >> 32)) : nan;
            if (a.dstTop) a.dstTop[i] = n ? (int64_t)index : -1;
            if (a.dstSamples) ((uint4*)a.dstSamples)[i] = n ? exportSample(a.items, a.numItems, index) : make_uint4(0, 0, 0, 0);
        }
    }
    nonempty = __reduce_add_sync(FULL, nonempty);
    if ((threadIdx.x & 31u) == 0 && nonempty) atomicAdd(&shNonempty, (unsigned long long)nonempty);
    __syncthreads();
    if (threadIdx.x == 0 && shNonempty) atomicAdd((unsigned long long*)&a.ctl->nonemptyCells, shNonempty);
}
