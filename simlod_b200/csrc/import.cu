// import.cu — octree import: a saved octree (simlod_load_octree, DESIGN.md §9.7) turned back into a live image, the
// Node / Chunk / OccupancyGrid image kernel_render, the exports and kernel_construct read, plus the builder's own side
// tables in the momentary buffer (construct_layout.cuh), so that the next kernel_construct launch continues as it would
// have in the context that saved the tree.
//
// The host has read and checked the records (a full export: breadth-first, consistent links and counts) and planned the
// heap: the root's grid at byte 16 as after a reset, one grid per other inner node, then every record's point chunks and
// voxel chunks, all lists in record order, so that chunk c of the plan holds the samples c covers in the file's order.
// Four launches and one per staged window:
//
//   simlod_import_nodes        one thread per record: nodes[i] = record i (children, level, X, Y, Z, name, counter,
//                              counts, list heads, grid) and its side-table entries; thread 0 the builder's control fields
//   simlod_import_link         one thread per chunk: its `next` link, and the chunk row entry of a point chunk
//   simlod_import_clear_grids  the grids, zeroed with 128-bit stores
//   simlod_import_scatter      per window of samples in device memory: one warp per chunk segment (<= 1000 samples),
//                              16-byte coalesced loads from the window, 16-byte stores into the chunk. A point must
//                              descend, by the builder's quantisation, to the leaf that holds it, and sets its cell in
//                              the grid of every node above it (warp-aggregated atomicOr): the grids are rebuilt from
//                              the points, by the builder's integer cells, as the builder's sampling built them
//   simlod_import_voxels       after the last window, three passes over the voxel chunks: every voxel is the centre of an
//                              occupied cell of its node; a voxel whose centre is one cell's only flips that cell's bit
//                              (a bit found flipped is a second voxel in the cell), and a second flip restores the grid
//   simlod_import_count_grids  one warp per grid: as many occupied cells as voxels (a split root: at most as many)
//
// Violations go to one error word the host reads once per load.
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "fpmath.cuh"
#include "construct_layout.cuh"
#include "kernel_args.h"

constexpr uint32_t PPC = SIMLOD_POINTS_PER_CHUNK;

__device__ __forceinline__ uint32_t ceilChunks(uint32_t n) { return (n + PPC - 1) / PPC; }
template <typename T> __device__ __forceinline__ T* table(const ImportArgs& a, uint64_t off) { return reinterpret_cast<T*>(a.scratch + off); }

extern "C" __global__ void __launch_bounds__(256)
simlod_import_nodes(const ImportArgs a) {
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid == 0) {                       // what kernel_construct initialises for a fresh tree (batchletIndex == 0)
        Ctl* ctl = table<Ctl>(a, scratch::OFF_CTL);
        ctl->errorFlags = 0;
        ctl->spilledTotal = 0; ctl->voxelsTotal = 0; ctl->voxelsByPass[0] = 0; ctl->voxelsByPass[1] = 0;
        for (int i = 0; i < 8; i++) ctl->phaseNanos[i] = 0;
        for (int i = 0; i < 16; i++) ctl->subNanos[i] = 0;
        ctl->launchCount = 0;
        for (int i = 0; i < 4; i++) ctl->events[i] = 0;
        for (int i = 0; i < 12; i++) for (int j = 0; j < 4; j++) ctl->roundHist[i][j] = 0;
        ctl->rowBump = a.numRows;         // every row is in use: no free rows
        ctl->rowFreeCount = 0;
    }
    for (uint32_t i = gid; i < a.numRecords; i += gridDim.x * blockDim.x) {
        const SimlodExportNode r = a.rec[i];
        const ImportPlan p = a.plan[i];
        SimlodNode* node = a.nodes + i;
        const bool inner = r.first_child >= 0;
        if (inner)
            for (int k = 0; k < 8; k++) node->children[k] = a.nodes + r.first_child + k;
        node->counter = p.counter;
        node->numPoints = r.num_points;
        node->level = r.level; node->X = r.X; node->Y = r.Y; node->Z = r.Z;
        for (int k = 0; k < 20; k++) node->name[k] = r.name[k];
        // a level-20 node's digit lies past the 20-byte name, where the builder writes it (on `visible`)
        if (r.level == SIMLOD_MAX_DEPTH) node->visible = (uint8_t)('0' + (((r.X & 1u) << 2) | ((r.Y & 1u) << 1) | (r.Z & 1u)));
        node->isLeaf = i == 0 ? 0 : 1;    // the root's stays as the reset leaves it
        const uint64_t grid = p.grid ? (uint64_t)(a.heap + p.grid) : 0ull;
        node->grid = reinterpret_cast<SimlodOccupancyGrid*>(grid);
        const uint32_t npc = ceilChunks(r.num_points), nvc = ceilChunks(r.num_voxels);
        const uint64_t first = (uint64_t)(a.heap + a.chunkBase) + p.chunk * SIMLOD_CHUNK_STRIDE;
        node->points = reinterpret_cast<SimlodChunk*>(npc ? first : 0ull);
        node->voxelChunks = reinterpret_cast<SimlodChunk*>(nvc ? first + (uint64_t)npc * SIMLOD_CHUNK_STRIDE : 0ull);
        node->numVoxels = r.num_voxels;
        node->numVoxelsStored = r.num_voxels;
        // the builder's side tables (construct.cu: split, allocateChunks, the launch prologue)
        table<uint32_t>(a, scratch::OFF_FIRSTCHILD)[i] = inner ? (uint32_t)r.first_child : 0u;
        table<uint32_t>(a, scratch::OFF_PARENT)[i] = r.parent >= 0 ? (uint32_t)r.parent : 0u;
        table<uint64_t>(a, scratch::OFF_GRIDPTR)[i] = grid;
        table<uint32_t>(a, scratch::OFF_LEAFROW)[i] = p.row;
        table<uint32_t>(a, scratch::OFF_SPLITSTATE)[i] = 0;
        table<uint64_t>(a, scratch::OFF_VTAIL)[i] = nvc ? first + (uint64_t)(npc + nvc - 1) * SIMLOD_CHUNK_STRIDE : 0ull;
        table<DirEntry>(a, scratch::OFF_VDIR)[i] = DirEntry{0, 0};
    }
}

// the record that owns chunk c: the last r with plan[r].chunk <= c (plan[numRecords].chunk is the total)
__device__ __forceinline__ uint32_t recordOf(const ImportArgs& a, uint64_t c) {
    uint32_t lo = 0, hi = a.numRecords;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a.plan[mid].chunk <= c) lo = mid; else hi = mid;
    }
    return lo;
}

extern "C" __global__ void __launch_bounds__(256)
simlod_import_link(const ImportArgs a, uint64_t numChunks) {
    for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < numChunks; c += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = recordOf(a, c);
        const SimlodExportNode& rec = a.rec[r];
        const ImportPlan& p = a.plan[r];
        const uint32_t npc = ceilChunks(rec.num_points), nvc = ceilChunks(rec.num_voxels);
        const uint32_t k = (uint32_t)(c - p.chunk);
        SimlodChunk* chunk = reinterpret_cast<SimlodChunk*>(a.heap + a.chunkBase + c * SIMLOD_CHUNK_STRIDE);
        const bool last = k + 1 == npc || k + 1 == npc + nvc;          // the last chunk of the point or the voxel list
        chunk->next = last ? nullptr : reinterpret_cast<SimlodChunk*>((uint8_t*)chunk + SIMLOD_CHUNK_STRIDE);
        if (k < npc) table<uint64_t>(a, scratch::OFF_ROWS)[(uint64_t)(p.row - 1) * scratch::ROW_SLOTS + k] = (uint64_t)chunk;
    }
}

// the root's grid at heap byte 16, then `numGrids` grids from `gridBase` on
extern "C" __global__ void __launch_bounds__(256)
simlod_import_clear_grids(uint8_t* heap, uint64_t gridBase, uint32_t numGrids) {
    constexpr uint64_t PER = SIMLOD_GRID_WORDS / 4;
    const uint64_t total = (uint64_t)(numGrids + 1) * PER;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t g = i / PER, w = i % PER;
        uint4* grid = reinterpret_cast<uint4*>(heap + (g == 0 ? 16 : gridBase + (g - 1) * SIMLOD_GRID_STRIDE));
        grid[w] = make_uint4(0, 0, 0, 0);
    }
}

// the cell of the point at `level` (construct.cu cellAt: bits [21 - level, 28 - level) of the 2^28 quantisation)
__device__ __forceinline__ uint32_t cellAtLevel(uint32_t pX, uint32_t pY, uint32_t pZ, uint32_t level) {
    const uint32_t sh = SIMLOD_MAX_DEPTH + 1 - level;
    return ((pX >> sh) & 127u) | (((pY >> sh) & 127u) << 7) | (((pZ >> sh) & 127u) << 14);
}

extern "C" __global__ void __launch_bounds__(256)
simlod_import_scatter(const ImportArgs a, const uint4* __restrict__ window, uint64_t winBegin, uint64_t winEnd, uint64_t chunk0, uint64_t chunk1) {
    const uint32_t FULL = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t numWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    // the octree cube as kernel_construct derives it from the box (construct.cu, launch prologue)
    const float size = fmaxf(fmaxf(fpx::sub(a.boxMax[0], a.boxMin[0]), fpx::sub(a.boxMax[1], a.boxMin[1])), fpx::sub(a.boxMax[2], a.boxMin[2]));
    const float rcpSize = fpx::rcp(size);
    uint32_t err = 0;
    for (uint64_t c = chunk0 + warp; c < chunk1; c += numWarps) {
        const uint32_t r = recordOf(a, c);
        const SimlodExportNode& rec = a.rec[r];
        const uint32_t np = rec.num_points, nv = rec.num_voxels, npc = ceilChunks(np);
        const uint32_t k = (uint32_t)(c - a.plan[r].chunk);
        const bool voxel = k >= npc;
        const uint64_t first = rec.sample_offset + (voxel ? np + (uint64_t)(k - npc) * PPC : (uint64_t)k * PPC);
        const uint32_t count = min(PPC, voxel ? nv - (k - npc) * PPC : np - k * PPC);
        const uint64_t lo = max(first, winBegin), hi = min(first + count, winEnd);
        if (lo >= hi) continue;
        const uint4* src = window + (lo - winBegin);
        uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<SimlodChunk*>(a.heap + a.chunkBase + c * SIMLOD_CHUNK_STRIDE)->points + (lo - first));
        const uint32_t n = (uint32_t)(hi - lo);
        const uint32_t shift = SIMLOD_MAX_DEPTH - rec.level;
        for (uint32_t base = 0; base < n; base += 32) {                 // warp-uniform trip count
            const uint32_t j = base + lane;
            const bool valid = j < n;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (valid) { v = __ldcs(src + j); dst[j] = v; }
            if (!voxel) {
                // construct.cu quantize(): X = u32(2^20 * (p - min) / size), pX = u32(2^28 * (p - min) / size)
                const float dx = fpx::add(__uint_as_float(v.x), -a.boxMin[0]);
                const float dy = fpx::add(__uint_as_float(v.y), -a.boxMin[1]);
                const float dz = fpx::add(__uint_as_float(v.z), -a.boxMin[2]);
                const uint32_t X = fpx::f2u(fpx::mul_ftz(fpx::mul(dx, 1048576.0f), rcpSize));
                const uint32_t Y = fpx::f2u(fpx::mul_ftz(fpx::mul(dy, 1048576.0f), rcpSize));
                const uint32_t Z = fpx::f2u(fpx::mul_ftz(fpx::mul(dz, 1048576.0f), rcpSize));
                const uint32_t pX = fpx::f2u(fpx::mul_ftz(fpx::mul(dx, 268435456.0f), rcpSize));
                const uint32_t pY = fpx::f2u(fpx::mul_ftz(fpx::mul(dy, 268435456.0f), rcpSize));
                const uint32_t pZ = fpx::f2u(fpx::mul_ftz(fpx::mul(dz, 268435456.0f), rcpSize));
                if (valid && (((X & 0xfffffu) >> shift) != rec.X || ((Y & 0xfffffu) >> shift) != rec.Y || ((Z & 0xfffffu) >> shift) != rec.Z))
                    err |= IMPORT_ERR_POINT;
                // the occupancy grids: every point sets its cell in each node it passed through, the inner nodes above
                // its leaf (and the root's grid while the root is a leaf), by the integer quantisation the builder
                // samples with. A grid is thus rebuilt from the points, never from the voxels' floats, whose cell
                // centres need not be distinct floats. Warp-aggregated: the lanes share the leaf and so the path.
                for (uint32_t node = r == 0 ? 0u : (uint32_t)rec.parent;;) {
                    const SimlodExportNode& an = a.rec[node];
                    uint32_t* grid = reinterpret_cast<uint32_t*>(a.heap + a.plan[node].grid);
                    const uint32_t cell = cellAtLevel(pX, pY, pZ, an.level);
                    const uint32_t wordKey = valid ? cell >> 5 : 0x80000000u | lane;     // lanes without a point: no word
                    const uint32_t peers = __match_any_sync(FULL, wordKey);
                    const uint32_t bits = __reduce_or_sync(peers, valid ? 1u << (cell & 31u) : 0u);
                    if (valid && lane == (uint32_t)(__ffs(peers) - 1)) atomicOr(&grid[cell >> 5], bits);
                    if (node == 0) break;
                    node = (uint32_t)an.parent;
                }
            }
        }
    }
    if (err) atomicOr(a.error, err);
}

// a voxel's cell centre along one axis by the builder's sequence (insertVoxel, construct.cu)
__device__ __forceinline__ float cellCentre(float base, float nodeSize, uint32_t c) {
    return fpx::add(base, fpx::mul_ftz(fpx::mul(nodeSize, fpx::add(fpx::u2f(c), 0.5f)), 0.0078125f));
}
// the cells [lo, hi] of one axis whose centre is bit for bit v (the centres are non-decreasing in the cell index; far
// from the box's origin, or deep in the tree, neighbouring cells can share one float); lo > hi if none
__device__ __forceinline__ void cellRange(float v, float base, float nodeSize, int32_t& lo, int32_t& hi) {
    uint32_t l = 0, h = 128;
    while (l < h) { const uint32_t m = (l + h) >> 1; if (cellCentre(base, nodeSize, m) < v) l = m + 1; else h = m; }
    lo = (int32_t)l;
    h = 128;
    while (l < h) { const uint32_t m = (l + h) >> 1; if (cellCentre(base, nodeSize, m) <= v) l = m + 1; else h = m; }
    hi = (int32_t)l - 1;
    if (lo <= hi && __float_as_uint(cellCentre(base, nodeSize, (uint32_t)lo)) != __float_as_uint(v)) hi = lo - 1;
}

// After every window: the voxels, read back from their chunks, against the grids the points rebuilt.
//   mode 0  every voxel is the centre of a cell whose bit is set
//   mode 1  a voxel whose centre belongs to one cell only flips that cell's bit; finding it already flipped is a second
//           voxel in that cell (not in the root once it has split: its list holds its pre-split voxels and their
//           re-creations, DESIGN.md §4)
//   mode 2  the same flips again, which restores the grids
extern "C" __global__ void __launch_bounds__(256)
simlod_import_voxels(const ImportArgs a, uint64_t numChunks, uint32_t mode) {
    const float size = fmaxf(fmaxf(fpx::sub(a.boxMax[0], a.boxMin[0]), fpx::sub(a.boxMax[1], a.boxMin[1])), fpx::sub(a.boxMax[2], a.boxMin[2]));
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t numWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    uint32_t err = 0;
    for (uint64_t c = warp; c < numChunks; c += numWarps) {
        const uint32_t r = recordOf(a, c);
        const SimlodExportNode& rec = a.rec[r];
        const uint32_t npc = ceilChunks(rec.num_points);
        const uint32_t k = (uint32_t)(c - a.plan[r].chunk);
        if (k < npc) continue;
        if (mode != 0 && r == 0 && rec.first_child >= 0) continue;
        const uint32_t count = min(PPC, rec.num_voxels - (k - npc) * PPC);
        const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const SimlodChunk*>(a.heap + a.chunkBase + c * SIMLOD_CHUNK_STRIDE)->points);
        uint32_t* grid = reinterpret_cast<uint32_t*>(a.heap + a.plan[r].grid);
        const float nodeSize = fpx::mul_ftz(fpx::ex2(-fpx::u2f(rec.level)), size);
        const float bx = fpx::fma(nodeSize, fpx::u2f(rec.X), a.boxMin[0]);
        const float by = fpx::fma(nodeSize, fpx::u2f(rec.Y), a.boxMin[1]);
        const float bz = fpx::fma(nodeSize, fpx::u2f(rec.Z), a.boxMin[2]);
        for (uint32_t j = lane; j < count; j += 32) {
            const uint4 v = src[j];
            int32_t x0, x1, y0, y1, z0, z1;
            cellRange(__uint_as_float(v.x), bx, nodeSize, x0, x1);
            cellRange(__uint_as_float(v.y), by, nodeSize, y0, y1);
            cellRange(__uint_as_float(v.z), bz, nodeSize, z0, z1);
            if (x0 > x1 || y0 > y1 || z0 > z1) { err |= IMPORT_ERR_VOXEL; continue; }
            if (mode == 0) {
                bool found = false;
                for (int32_t cz = z0; cz <= z1 && !found; cz++)
                    for (int32_t cy = y0; cy <= y1 && !found; cy++)
                        for (int32_t cx = x0; cx <= x1 && !found; cx++) {
                            const uint32_t cell = (uint32_t)cx | ((uint32_t)cy << 7) | ((uint32_t)cz << 14);
                            found = (grid[cell >> 5] >> (cell & 31u)) & 1u;
                        }
                if (!found) err |= IMPORT_ERR_VOXEL;
            } else if (x0 == x1 && y0 == y1 && z0 == z1) {
                const uint32_t cell = (uint32_t)x0 | ((uint32_t)y0 << 7) | ((uint32_t)z0 << 14), bit = 1u << (cell & 31u);
                const uint32_t old = atomicXor(&grid[cell >> 5], bit);
                if (mode == 1 && !(old & bit)) err |= IMPORT_ERR_DUPLICATE;
            }
        }
    }
    if (err) atomicOr(a.error, err);
}

// one warp per record with a grid: the occupied cells against the voxels, equal everywhere but in a root that has split
// (there the pre-split voxels come on top, DESIGN.md §4)
extern "C" __global__ void __launch_bounds__(256)
simlod_import_count_grids(const ImportArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, numWarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t r = warp; r < a.numRecords; r += numWarps) {
        if (a.plan[r].grid == 0) continue;
        const uint4* g = reinterpret_cast<const uint4*>(a.heap + a.plan[r].grid);
        uint32_t n = 0;
        for (uint32_t i = lane; i < SIMLOD_GRID_WORDS / 4; i += 32) { const uint4 w = g[i]; n += __popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w); }
        n = __reduce_add_sync(0xffffffffu, n);
        const uint32_t nv = a.rec[r].num_voxels;
        const bool ok = (r == 0 && a.rec[r].first_child >= 0) ? n <= nv : n == nv;
        if (lane == 0 && !ok) atomicOr(a.error, (uint32_t)IMPORT_ERR_COUNT);
    }
}
