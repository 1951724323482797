// export.cu — octree export: the node hierarchy and its samples as flat arrays (DESIGN.md §9.4), whole, cut at one
// depth, or the LOD cut one camera sees (§9.5).
//
// Reads the ABI only (Node::children, points / numPoints, voxelChunks / numVoxelsStored, the heap header and
// Stats::numNodes; for the view also the fields the renderer's cut reads), so an octree built by the reference kernels
// exports exactly like ours. Three launches, four for the view:
//
//   simlod_export_view_flags  (view only) one thread per node of nodes[]: whether kernel_render would draw it for the
//                          uniforms, by the renderer's own test (nodeDrawn, lodcut.cuh), as one byte per node index
//   simlod_export_plan     one block: breadth-first order level by level from the root (records in (level, Morton) order,
//                          the 8 children of a node consecutive), per-record sample counts, the exclusive scans that give
//                          sample_offset and each list's first chunk item, and ExportCtl (sizes + error);
//                          simlod_export_plan_view, the view's instance of the same code, cuts the breadth-first records
//                          down to the paths that reach the drawn nodes
//   simlod_export_collect  one thread per sampled record walks its chunk lists (the dependent ->next chains), tests every
//                          pointer before it dereferences it and writes one item per chunk: source chunk, destination
//                          index, count
//   simlod_export_gather   after the host has checked ExportCtl: warps copy the node records, then pop chunk items
//                          (<= 1000 samples each) and copy them with 16-byte loads and coalesced streaming stores
//
// The octree file (simlod_save_octree, DESIGN.md §9.7) runs the full plan and collect, then simlod_export_counters (the
// records' Node::counter) and simlod_export_gather_window, the gather's instance that copies one bounded window of the
// sample array at a time.
//
// The flags, plan and collect kernels write scratch and ExportCtl only; nothing reaches the destination before the
// gather. Nothing is written into nodes[] (not even the visible / isLarge flags kernel_render stores there).
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "lodcut.cuh"
#include "export_common.cuh"

// One thread per node of nodes[]: drawn[n] = whether kernel_render draws node n for the uniforms `u`, by the renderer's own
// test (lodcut.cuh). The uniforms come by value, as kernel_render receives them. Writes nothing into nodes[].
extern "C" __global__ void __launch_bounds__(256)
simlod_export_view_flags(const SimlodNode* __restrict__ nodes, const SimlodStats* __restrict__ stats, const SimlodUniforms u,
                         uint32_t maxRecords, uint8_t* __restrict__ drawn) {
    const uint32_t numNodes = min(stats->numNodes, maxRecords);        // more nodes than records: the plan reports it
    const float cubeSize = cubeSizeOf(u);
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < numNodes; n += gridDim.x * blockDim.x) {
        bool visible, large;
        drawn[n] = nodeDrawn(u, nodes + n, cubeSize, u.boxMin[0], u.boxMin[1], u.boxMin[2], visible, large) ? 1 : 0;
    }
}

// depth < 0: full export. Scratch: rec[maxRecords] (SimlodExportNode), recNode[maxRecords] (node index),
// recItem[maxRecords] (first chunk item of the record's point list; its voxel list follows).
// isView: the view export (depth < 0, view.drawn set). The breadth-first pass covers every reachable node (so an
// inconsistent image is reported wherever it is), a record is sampled when its node is drawn, and the records kept are
// the root and the 8 children of every record with a drawn record strictly below it. A template parameter rather than a
// test of view.drawn, so that the full and depth exports compile to the plan they had before the view existed.
template <bool isView>
__device__ __forceinline__ void plan(const uint8_t* __restrict__ nodes, const SimlodStats* __restrict__ stats, int32_t depth,
                                     uint32_t maxRecords, SimlodExportNode* __restrict__ rec, uint32_t* __restrict__ recNode,
                                     uint64_t* __restrict__ recItem, ExportCtl* __restrict__ ctl, const ViewScratch& view) {
    __shared__ uint32_t sh_total, sh_error, sh_maxLevel;
    const uint32_t numNodes = stats->numNodes;
    const uint64_t nodesAddr = (uint64_t)nodes;
    SimlodExportNode* const bRec = isView ? view.rec : rec;           // breadth-first records
    uint32_t* const bNode = isView ? view.recNode : recNode;
    if (threadIdx.x == 0) {
        sh_total = 1; sh_error = 0; sh_maxLevel = 0;
        if (numNodes == 0 || numNodes > maxRecords) sh_error = EXPORT_ERR_CHILD;
        bNode[0] = 0;
        bRec[0].parent = -1;
    }
    __syncthreads();
    if (sh_error) { if (threadIdx.x == 0) ctl->error = sh_error; return; }

    // deepest level in the octree: every allocated node
    uint32_t lmax = 0;
    for (uint32_t i = threadIdx.x; i < numNodes; i += PLAN_THREADS)
        lmax = max(lmax, ((const SimlodNode*)(nodes + (uint64_t)i * sizeof(SimlodNode)))->level);
    atomicMax(&sh_maxLevel, lmax);

    // breadth-first, level by level: the children of the records [begin, end) are appended in record order, 8 per inner
    // node in child-index order, which is (level, Morton) order one level down
    uint32_t begin = 0, end = 1;
    for (int32_t level = 0; begin < end; level++) {
        const bool expand = depth < 0 || level < depth;
        for (uint32_t tile = begin; tile < end; tile += PLAN_THREADS) {
            const uint32_t r = tile + threadIdx.x;
            const bool valid = r < end;
            uint32_t numChildren = 0, err = 0;
            uint64_t child[8];
            const SimlodNode* node = nullptr;
            if (valid) {
                node = (const SimlodNode*)(nodes + (uint64_t)bNode[r] * sizeof(SimlodNode));
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
            const uint32_t pos = (uint32_t)blockScan<isView>(valid && expand && inner && !err ? 8 : 0, &total);
            const uint32_t first = sh_total + pos;
            __syncthreads();
            if (threadIdx.x == 0) {
                if (sh_total + total > numNodes) atomicMax(&sh_error, EXPORT_ERR_CHILD);   // more records than nodes
                else sh_total += (uint32_t)total;
            }
            if (err) atomicMax(&sh_error, err);
            if (valid) {
                const bool addChildren = expand && inner && !err && first + 8 <= numNodes;
                if (addChildren) {
                    #pragma unroll
                    for (int k = 0; k < 8; k++) {
                        bNode[first + k] = (uint32_t)((child[k] - nodesAddr) / sizeof(SimlodNode));
                        bRec[first + k].parent = (int32_t)r;
                    }
                }
                // what this record contributes: everything (full), the voxels of an inner node at the cut level, the
                // points of a leaf at or above it; for the view, both lists of a drawn node and nothing else
                const uint32_t np = node->numPoints, nv = node->numVoxelsStored;
                const bool full = depth < 0;
                const bool sampled = isView ? view.drawn[bNode[r]] != 0 : full || !inner || level == depth;
                SimlodExportNode& o = bRec[r];
                o.level = node->level; o.X = node->X; o.Y = node->Y; o.Z = node->Z;
                const uint32_t* nm = (const uint32_t*)node->name;
                uint32_t* onm = (uint32_t*)o.name;
                #pragma unroll
                for (int k = 0; k < 5; k++) onm[k] = nm[k];
                o.flags = (inner ? 0u : (uint32_t)SIMLOD_EXPORT_LEAF) | (sampled ? (uint32_t)SIMLOD_EXPORT_SAMPLED : 0u);
                o.first_child = addChildren ? (int32_t)first : -1;
                o.num_points = (!isView || sampled) && (full || !inner) ? np : 0;
                o.num_voxels = (!isView || sampled) && (full || (inner && level == depth)) ? nv : 0;
            }
            __syncthreads();
            if (sh_error) break;
        }
        if (sh_error) break;
        begin = end;
        end = sh_total;
    }
    __syncthreads();
    if (sh_error) { if (threadIdx.x == 0) ctl->error = sh_error; return; }

    uint32_t n = sh_total;
    if (isView) {
        // |D|: the nodes of nodes[] the renderer draws
        uint32_t numDrawn = 0;
        for (uint32_t i = threadIdx.x; i < numNodes; i += PLAN_THREADS) numDrawn += view.drawn[i];
        uint64_t drawnTotal = 0;
        blockScan<isView>(numDrawn, &drawnTotal);
        // mark the ancestors of every drawn record, walking up the parent links (parents precede their children, so a
        // walk ends at the root within 20 steps). The stores are idempotent; a walk stops at a record another thread has
        // marked, since that thread goes on to the root.
        for (uint32_t r = threadIdx.x; r < n; r += PLAN_THREADS) view.mark[r] = 0;
        __syncthreads();
        for (uint32_t r = threadIdx.x; r < n; r += PLAN_THREADS)
            if (view.rec[r].flags & SIMLOD_EXPORT_SAMPLED)
                for (int32_t p = view.rec[r].parent; p >= 0 && !view.mark[p]; p = view.rec[p].parent) view.mark[p] = 1;
        __syncthreads();
        // keep the root and every child of a marked record: whole sibling groups, in breadth-first order. Every drawn
        // record's parent is marked, so all of them are kept; a drawn node the pass did not reach (or reached twice)
        // shows as a count other than |D|.
        uint32_t kept = 0, keptDrawn = 0;
        for (uint32_t tile = 0; tile < n; tile += PLAN_THREADS) {
            const uint32_t r = tile + threadIdx.x;
            bool keep = false;
            if (r < n) { const int32_t p = view.rec[r].parent; keep = p < 0 || view.mark[p]; }
            uint64_t total = 0;
            const uint32_t pos = (uint32_t)blockScan<isView>(keep ? 1 : 0, &total);
            if (keep) view.index[r] = kept + pos;
            kept += (uint32_t)total;
            keptDrawn += (uint32_t)__syncthreads_count(keep && (view.rec[r].flags & SIMLOD_EXPORT_SAMPLED));
        }
        if (keptDrawn != drawnTotal) { if (threadIdx.x == 0) ctl->error = EXPORT_ERR_CHILD; return; }
        // the kept records at their positions, parent and first_child remapped (first_child only on marked records)
        for (uint32_t r = threadIdx.x; r < n; r += PLAN_THREADS) {
            const int32_t p = view.rec[r].parent;
            if (p >= 0 && !view.mark[p]) continue;
            SimlodExportNode o = view.rec[r];
            o.parent = p < 0 ? -1 : (int32_t)view.index[p];
            o.first_child = view.mark[r] ? (int32_t)view.index[o.first_child] : -1;
            const uint32_t k = view.index[r];
            rec[k] = o;
            recNode[k] = view.recNode[r];
        }
        n = kept;
        __syncthreads();
    }

    // sample offsets and chunk items: exclusive scans over the records
    uint64_t samplesBase = 0, itemsBase = 0, points = 0, voxels = 0;
    for (uint32_t tile = 0; tile < n; tile += PLAN_THREADS) {
        const uint32_t r = tile + threadIdx.x;
        uint32_t np = 0, nv = 0;
        if (r < n) { np = rec[r].num_points; nv = rec[r].num_voxels; }
        uint64_t tS = 0, tI = 0, tP = 0, tV = 0;
        const uint64_t s = blockScan<isView>((uint64_t)np + nv, &tS);
        const uint64_t it = blockScan<isView>(ceilChunks(np) + ceilChunks(nv), &tI);
        blockScan<isView>(np, &tP);
        blockScan<isView>(nv, &tV);
        if (r < n) { rec[r].sample_offset = samplesBase + s; recItem[r] = itemsBase + it; }
        samplesBase += tS; itemsBase += tI; points += tP; voxels += tV;
    }
    if (threadIdx.x == 0) {
        ctl->numNodes = n; ctl->maxLevel = sh_maxLevel;
        ctl->numSamples = samplesBase; ctl->numPoints = points; ctl->numVoxels = voxels;
        ctl->numItems = itemsBase; ctl->error = 0;
    }
}

extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_export_plan(const uint8_t* __restrict__ nodes, const SimlodStats* __restrict__ stats, int32_t depth, uint32_t maxRecords,
                   SimlodExportNode* __restrict__ rec, uint32_t* __restrict__ recNode, uint64_t* __restrict__ recItem,
                   ExportCtl* __restrict__ ctl) {
    plan<false>(nodes, stats, depth, maxRecords, rec, recNode, recItem, ctl, ViewScratch{});
}

// the plan of the view export: depth < 0, the drawn flags of simlod_export_view_flags in view.drawn
extern "C" __global__ void __launch_bounds__(PLAN_THREADS)
simlod_export_plan_view(const uint8_t* __restrict__ nodes, const SimlodStats* __restrict__ stats, uint32_t maxRecords,
                        SimlodExportNode* __restrict__ rec, uint32_t* __restrict__ recNode, uint64_t* __restrict__ recItem,
                        ExportCtl* __restrict__ ctl, const ViewScratch view) {
    plan<true>(nodes, stats, -1, maxRecords, rec, recNode, recItem, ctl, view);
}

// Walks `count` samples' worth of chunks of the list at `head`. Every chunk must lie inside the used heap
// [heap, heap + heapUsed) and be 16-byte aligned before it is read; the list must not end early.
__device__ __forceinline__ uint32_t walkList(uint64_t head, uint32_t count, uint64_t heap, uint64_t heapUsed, uint64_t dst,
                                             Item* __restrict__ items) {
    uint64_t addr = head;
    for (uint32_t c = 0; c < ceilChunks(count); c++) {
        if (addr == 0) return EXPORT_ERR_SHORT;
        if (addr < heap || addr - heap > heapUsed || heapUsed - (addr - heap) < sizeof(SimlodChunk) || (addr - heap) % 16 != 0)
            return EXPORT_ERR_CHUNK;
        const uint32_t take = min(count - c * PPC, PPC);
        items[c] = Item{addr, (dst + (uint64_t)c * PPC) | ((uint64_t)take << 48)};
        addr = (uint64_t)((const SimlodChunk*)addr)->next;
    }
    return 0;
}

extern "C" __global__ void __launch_bounds__(256)
simlod_export_collect(const uint8_t* __restrict__ nodes, const uint8_t* __restrict__ heap, uint64_t heapBytes,
                      const SimlodExportNode* __restrict__ rec, const uint32_t* __restrict__ recNode, const uint64_t* __restrict__ recItem,
                      Item* __restrict__ items, uint64_t itemsCap, ExportCtl* __restrict__ ctl) {
    if (ctl->error) return;
    // more chunks than the used heap can hold: the counts do not match the lists (the scratch holds one item per chunk)
    if (ctl->numItems > itemsCap) { if (blockIdx.x == 0 && threadIdx.x == 0) atomicMax(&ctl->error, (uint32_t)EXPORT_ERR_SHORT); return; }
    const uint32_t n = ctl->numNodes;
    const uint64_t heapAddr = (uint64_t)heap;
    const uint64_t heapUsed = min(((const SimlodHeapHeader*)heap)->offset, heapBytes);
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        const uint32_t np = rec[r].num_points, nv = rec[r].num_voxels;
        if (np == 0 && nv == 0) continue;
        const SimlodNode* node = (const SimlodNode*)(nodes + (uint64_t)recNode[r] * sizeof(SimlodNode));
        const uint64_t base = recItem[r], dst = rec[r].sample_offset;
        uint32_t err = walkList((uint64_t)node->points, np, heapAddr, heapUsed, dst, items + base);
        if (!err) err = walkList((uint64_t)node->voxelChunks, nv, heapAddr, heapUsed, dst + np, items + base + ceilChunks(np));
        if (err) atomicMax(&ctl->error, err);
    }
}

constexpr uint32_t GATHER_UNROLL = 8;

// windowed: the octree file's staging (simlod_save_octree) — no records, and of every item only the samples whose
// destination index lies in [winBegin, winEnd), written at index - winBegin. A template parameter, so that the export's
// own gather compiles to the kernel it was before the window existed.
template <bool windowed>
__device__ __forceinline__ void gather(const uint4* __restrict__ rec, uint4* __restrict__ dstNodes, const Item* __restrict__ items,
                                       uint4* __restrict__ dstSamples, const ExportCtl* __restrict__ ctl, uint64_t winBegin, uint64_t winEnd) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t numWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    if (!windowed) {
        const uint64_t recWords = (uint64_t)ctl->numNodes * (sizeof(SimlodExportNode) / 16);
        for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < recWords; i += (uint64_t)gridDim.x * blockDim.x)
            __stcs(dstNodes + i, rec[i]);
    }
    const uint64_t numItems = ctl->numItems;
    for (uint64_t k = warp; k < numItems; k += numWarps) {
        const Item it = items[k];
        const uint4* __restrict__ src = (const uint4*)it.src;
        uint4* __restrict__ dst = dstSamples + (it.dst & 0xffffffffffffull);
        uint32_t count = (uint32_t)(it.dst >> 48);
        if (windowed) {
            const uint64_t d0 = it.dst & 0xffffffffffffull;
            const uint64_t lo = max(d0, winBegin), hi = min(d0 + count, winEnd);
            if (lo >= hi) continue;
            src += lo - d0;
            dst = dstSamples + (lo - winBegin);
            count = (uint32_t)(hi - lo);
        }
        for (uint32_t b = 0; b < count; b += 32 * GATHER_UNROLL) {
            uint4 v[GATHER_UNROLL];
            #pragma unroll
            for (uint32_t u = 0; u < GATHER_UNROLL; u++) {
                const uint32_t j = b + u * 32 + lane;
                if (j < count) v[u] = __ldcs(src + j);
            }
            #pragma unroll
            for (uint32_t u = 0; u < GATHER_UNROLL; u++) {
                const uint32_t j = b + u * 32 + lane;
                if (j < count) __stcs(dst + j, v[u]);
            }
        }
    }
}

extern "C" __global__ void __launch_bounds__(256)
simlod_export_gather(const uint4* __restrict__ rec, uint4* __restrict__ dstNodes, const Item* __restrict__ items,
                     uint4* __restrict__ dstSamples, const ExportCtl* __restrict__ ctl) {
    gather<false>(rec, dstNodes, items, dstSamples, ctl, 0, 0);
}

// The samples of the full export whose index lies in [winBegin, winEnd), into window[0, winEnd - winBegin)
extern "C" __global__ void __launch_bounds__(256)
simlod_export_gather_window(const Item* __restrict__ items, uint4* __restrict__ window, const ExportCtl* __restrict__ ctl,
                            uint64_t winBegin, uint64_t winEnd) {
    gather<true>(nullptr, nullptr, items, window, ctl, winBegin, winEnd);
}

// Node::counter of every record's node (the octree file's counters section; the records do not carry it)
extern "C" __global__ void __launch_bounds__(256)
simlod_export_counters(const SimlodNode* __restrict__ nodes, const uint32_t* __restrict__ recNode, const ExportCtl* __restrict__ ctl,
                       uint32_t* __restrict__ counters) {
    const uint32_t n = ctl->numNodes;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) counters[r] = nodes[recNode[r]].counter;
}
