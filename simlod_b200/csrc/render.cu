// render.cu — software point/voxel rasteriser for sm_90a (H100).
//
// Drop-in for the reference's `kernel_render` (modules/progressive_octree/render.cu:1084-1355):
// same extern "C" name and arguments, same outputs — Node::visible / Node::isLarge flags, the
// packed depth|colour u64 framebuffer at byte 31 200 144 of the render buffer, the RGBA8 surface,
// and Stats::numVisible* — bit for bit for the same octree buffers and Uniforms.
//
// What is different is the work decomposition. The reference assigns one 256-thread block per
// visible NODE (render.cu:181-207), so a 50 000-point leaf and a 200-voxel inner node cost one
// block each, and every thread re-walks the node's chunk list. Here the LOD cut emits
// CHUNK-granular work items (<= 1000 samples = 16 KB, contiguous), and persistent warps pull items
// from one queue with a single atomicAdd each, read samples with coalesced 128-bit loads, and
// splat with an early-out compare + 64-bit atomicMin (the 16.6 MB framebuffer stays L2-resident).
//
// Every floating-point value that decides a pixel or a visibility bit is computed with the exact
// instruction sequence the reference's SASS uses (see fpmath.cuh and DESIGN.md §5).
#include <cooperative_groups.h>
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "fpmath.cuh"
#include "lodcut.cuh"
#include "region.cuh"
#include "render_layout.cuh"
#include "splat.cuh"

namespace cg = cooperative_groups;

typedef SimlodPoint Point;
typedef SimlodChunk Chunk;
typedef SimlodNode Node;
typedef SimlodStats Stats;
typedef SimlodUniforms Uniforms;
typedef SimlodFloat4 Row;
struct CudaPrint;


// One work item = one chunk of <= 1000 samples, packed into a single 64-bit word:
//   [63:26] (chunk address - heap base) >> 4   [25:16] sample count (1..1000)   [15:11] node level   [10:4] node colour id   [0] valid
// ITEM_EMPTY = nothing to draw (list shorter than the counters say).
typedef uint64_t WorkItem;
constexpr WorkItem ITEM_EMPTY = ~0ull;
__device__ __forceinline__ WorkItem packItem(const uint8_t* heapBase, const void* chunk, uint32_t count, uint32_t level, uint32_t colorId) {
    return ((uint64_t)((const uint8_t*)chunk - heapBase) >> 4 << 26) | ((uint64_t)count << 16) | ((uint64_t)(level & 31u) << 11) | ((uint64_t)(colorId & 127u) << 4) | 1ull;
}
__device__ __forceinline__ const uint4* itemSamples(const uint8_t* heapBase, WorkItem w) { return reinterpret_cast<const uint4*>(heapBase + ((w >> 26) << 4)); }
__device__ __forceinline__ uint32_t itemCount(WorkItem w) { return (uint32_t)(w >> 16) & 1023u; }
__device__ __forceinline__ uint32_t itemLevel(WorkItem w) { return (uint32_t)(w >> 11) & 31u; }
__device__ __forceinline__ uint32_t itemColorId(WorkItem w) { return (uint32_t)(w >> 4) & 127u; }

struct RCtl {
    uint32_t numItems;
    uint32_t head[3];            // queue heads: single pass / HQS depth pass / HQS colour pass
    uint32_t numVisibleNodes, numVisiblePoints, numVisibleVoxels, numVisibleInner, numVisibleLeaves;
    uint32_t overflow;
    uint32_t cacheHits, cacheWalks;      // lists served from the chunk-list cache / walked (developer counters)
    uint64_t phaseNanos[6];              // @48 last frame, by the grid's first thread: clear|visibility+cut, -, items, draw (all passes), stats+EDL
    // The cut runs in the first phase of a frame, so its counter cannot be cleared at the start of that frame (no barrier
    // in between): the previous frame leaves it at 0 and says so with the magic next to it. A buffer that never saw a frame
    // of this kernel (or was scribbled over since: both words lie inside the reference's first Node copy) takes one
    // extra barrier. Nobody writes the magic before the last barrier of a frame, so all threads agree on what they read.
    uint32_t cutCount;                   // @96 drawn nodes of this frame
    uint32_t cutMagic;                   // @100
};
constexpr uint32_t CUT_MAGIC = 0xC07C0DE5u;
static_assert(offsetof(RCtl, cutCount) == 96 && offsetof(RCtl, cutMagic) == 100, "cutCount / cutMagic are one aligned 8-byte pair");
static_assert(offsetof(RCtl, cacheHits) == 40 && offsetof(RCtl, phaseNanos) == 48, "tools and tests read RCtl by offset");

// ---- chunk-list cache ---------------------------------------------------------------------------------------
// Chunk lists are singly linked, so the k-th chunk of a node is k dependent loads away; the reference makes every
// thread of a block walk the list (render.cu:116-121). Frames follow each other with the same nodes in view, so the
// chunk pointers of a drawn node are kept, per node and list, in the tail of the render buffer. A cached array is only
// a HINT: it is used after it has been verified against the octree — entry 0 is the list head and every chunk's `next`
// is the following entry — which takes independent loads (32 per warp step) instead of a dependent chain, and proves
// the array equals the list whatever happened in between (growth, a reset, another render kernel scribbling over
// the buffer). Pointers are range-checked against the heap before they are followed. A list that fails, or has grown,
// is walked (from the verified prefix on) and cached again.
struct ListEntry { uint32_t off, n, cap, pad; };           // pool[off .. off + n) = the first n chunks of the list; cap reserved
struct CacheHeader { uint32_t magic, cursor, poolCap, pad; };
constexpr uint32_t CACHE_MAGIC = 0x51D0CAC3u;

__device__ __forceinline__ uint32_t ldv(const uint32_t* p) { return *(volatile const uint32_t*)p; }
__device__ __forceinline__ uint32_t laneId() { return threadIdx.x & 31; }
__device__ __forceinline__ uint64_t globaltimer() { uint64_t t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

// One thread per node: the node's flags (render.cu:762-901) and, in the same phase, the LOD cut (render.cu:906-933), both
// from nodeDrawn (lodcut.cuh). A node is drawn when it is a visible non-large child of a large node, or a large visible
// leaf. The child recomputes its parent's `isLarge` instead of waiting for the thread that owns the parent: no barrier
// between the flags and the cut.
__device__ void computeVisibilityAndCut(const Uniforms& u, Node* nodes, uint32_t numNodes, float cubeSize,
                                        float cminx, float cminy, float cminz, RCtl* ctl, uint32_t* visList) {
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < numNodes; n += stride) {
        Node* node = &nodes[n];
        bool visible, large;
        const bool drawn = nodeDrawn(u, node, cubeSize, cminx, cminy, cminz, visible, large);
        node->visible = visible ? 1 : 0;
        node->isLarge = large ? 1 : 0;
        if (drawn) {
            uint32_t v = atomicAdd(&ctl->cutCount, 1u);
            if (v < rbuf::VIS_CAP) visList[v] = n;
        }
    }
}

// ------------------------------------------------------------------------------------------
// visibility, pass 2: LOD cut (render.cu:906-933), then the chunk items of every drawn node (a visible non-large
// child of a large node, or a large visible leaf): a whole warp turns the node's two chunk lists into work items
// through the cache above.
// ------------------------------------------------------------------------------------------
struct EmitCtx {
    RCtl* ctl;
    WorkItem* items;
    const Node* nodes;
    const uint8_t* heapBase;
    uint64_t heapUsed;           // bytes of the heap in use (AllocatorGlobal::offset): chunk pointers must lie below
    CacheHeader* cache;
    ListEntry* entries;          // [node][2]
    uint64_t* pool;
    uint32_t poolCap;            // 0: cache disabled (render buffer too small for this resolution)
};

__device__ __forceinline__ bool validChunkPointer(const EmitCtx& e, uint64_t p) {
    const uint64_t base = (uint64_t)e.heapBase;
    return p >= base + 16 && p + sizeof(Chunk) <= base + e.heapUsed && ((p - base) & 15ull) == 0;
}

// one chunk list of a drawn node -> n work items at items[0..n). Warp-cooperative (all 32 lanes).
__device__ void emitList(const EmitCtx& e, const Chunk* head, uint32_t n, uint32_t count, uint32_t level, uint32_t colorId, ListEntry* entry, WorkItem* items) {
    const uint32_t FULL = 0xffffffffu;
    const uint32_t lane = laneId();
    if (n == 0) return;
    auto samplesOf = [&](uint32_t k) { return k + 1 < n ? (uint32_t)SIMLOD_POINTS_PER_CHUNK : count - (n - 1) * SIMLOD_POINTS_PER_CHUNK; };

    ListEntry le = *entry;
    uint32_t m = 0;                                       // chunks of the list the cache claims to know
    if (e.poolCap != 0 && le.n != 0 && le.n <= le.cap && (uint64_t)le.off + le.cap <= e.poolCap) m = min(le.n, n);
    // ---- verify the cached prefix with independent loads, and emit it
    uint64_t carriedNext = 0;                             // `next` of the last verified chunk
    bool ok = true;
    for (uint32_t k0 = 0; k0 < m && ok; k0 += 32) {
        const uint32_t k = k0 + lane;
        const bool have = k < m;
        const uint64_t p = have ? e.pool[le.off + k] : 0ull;
        if (!__all_sync(FULL, !have || validChunkPointer(e, p))) { ok = false; break; }
        const uint64_t nx = have ? (uint64_t)reinterpret_cast<const Chunk*>(p)->next : 0ull;
        uint64_t nxPrev = __shfl_up_sync(FULL, nx, 1);
        if (lane == 0) nxPrev = carriedNext;
        const bool good = !have || (k == 0 ? p == (uint64_t)head : nxPrev == p);
        if (!__all_sync(FULL, good)) { ok = false; break; }
        const uint32_t lastLane = min(31u, m - 1 - k0);
        carriedNext = __shfl_sync(FULL, nx, lastLane);
        if (have) items[k] = packItem(e.heapBase, reinterpret_cast<const void*>(p), samplesOf(k), level, colorId);
    }
    if (!ok) m = 0;
    if (m == n) { if (lane == 0) atomicAdd(&e.ctl->cacheHits, 1u); return; }

    // ---- the rest of the list (all of it when nothing was cached, or the cache was wrong): a dependent walk by one lane.
    // The pointers go to the cache: in place while the reserved room lasts, else to a fresh, larger array.
    if (lane == 0) atomicAdd(&e.ctl->cacheWalks, 1u);
    uint32_t off = le.off, cap = le.cap;
    bool caching = e.poolCap != 0;
    if (caching && (m == 0 || n > cap)) {
        uint32_t want = n + max(8u, n / 4u);
        uint32_t at = 0;
        if (lane == 0) at = atomicAdd(&e.cache->cursor, want);
        at = __shfl_sync(FULL, at, 0);
        if ((uint64_t)at + want > e.poolCap) caching = false;            // pool exhausted: drawn without caching; the pool restarts next frame
        else {
            for (uint32_t k = lane; k < m; k += 32) e.pool[at + k] = e.pool[off + k];       // keep the verified prefix
            off = at; cap = want;
        }
    }
    __syncwarp();
    if (lane == 0) {
        const Chunk* cur = m == 0 ? head : reinterpret_cast<const Chunk*>(carriedNext);
        uint32_t k = m;
        for (; k < n; k++) {
            if (cur == nullptr || !validChunkPointer(e, (uint64_t)cur)) break;
            if (caching) e.pool[off + k] = (uint64_t)cur;
            items[k] = packItem(e.heapBase, cur, samplesOf(k), level, colorId);
            cur = cur->next;
        }
        const uint32_t known = k;
        for (; k < n; k++) items[k] = ITEM_EMPTY;
        if (caching) *entry = ListEntry{off, known, cap, 0};
    }
    __syncwarp();
}

__device__ void emitNode(const EmitCtx& e, const Node* node) {
    const uint32_t lane = laneId();
    const uint32_t numPoints = node->numPoints, numVoxels = node->numVoxels, level = node->level;
    const uint32_t nP = (numPoints + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
    const uint32_t nV = (numVoxels + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
    uint32_t base = 0;
    if (lane == 0) {                                                                 // render.cu:918-932 bookkeeping
        if (numPoints > 0) { atomicAdd(&e.ctl->numVisibleLeaves, 1u); atomicAdd(&e.ctl->numVisiblePoints, numPoints); }
        else if (numVoxels > 0) { atomicAdd(&e.ctl->numVisibleInner, 1u); atomicAdd(&e.ctl->numVisibleVoxels, numVoxels); }
        if (nP + nV) base = atomicAdd(&e.ctl->numItems, nP + nV);
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    if (nP + nV == 0) return;
    if ((uint64_t)base + nP + nV > rbuf::ITEM_CAP) { if (lane == 0) atomicOr(&e.ctl->overflow, 1u); return; }
    const uint32_t colorId = nodeColorId(node);
    const uint32_t index = (uint32_t)(node - e.nodes);
    emitList(e, node->points, nP, numPoints, level, colorId, &e.entries[2 * index + 0], e.items + base);
    emitList(e, node->voxelChunks, nV, numVoxels, level, colorId, &e.entries[2 * index + 1], e.items + base + nP);
}

// drawn nodes -> chunk items: one WARP per node, the nodes spread over all warps of the grid (drawn nodes cluster in
// nodes[]: the 8 children of a node are neighbours)
__device__ void emitVisible(const EmitCtx& e, const uint32_t* visList, uint32_t numVisible) {
    const uint32_t numWarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t warp = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;
    for (uint32_t v = warp; v < numVisible; v += numWarps) emitNode(e, &e.nodes[visList[v]]);
}

// one pass over the frame's items: every warp starts with the item of its own number (no atomic: 4 224 warps on an H100 popping the
// same counter at the same instant would serialise), then persistent warps pop the rest
// with a single atomicAdd each; a frame with no more items than warps touches the counter not at all.
// (Measured and rejected, profiles/r02/render_notes.md: quarter-chunk items, 2 / 4 warps per item on small frames, the next
// pop prefetched under the current item, four sample loads in flight per lane — each within 3 % of this loop or slower.)
template <typename F>
__device__ __forceinline__ void forEachSample(const uint8_t* heapBase, const WorkItem* items, uint32_t numItems, uint32_t* head, F&& f) {
    const uint32_t lane = laneId();
    const uint32_t numWarps = (gridDim.x * blockDim.x) >> 5;
    uint32_t it = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;       // neighbouring items (chunks of one node) go to different SMs
    while (it < numItems) {
        WorkItem w = items[it];
        if (w != ITEM_EMPTY && w != 0) {
            const uint4* pts = itemSamples(heapBase, w);
            const uint32_t count = itemCount(w), level = itemLevel(w), colorId = itemColorId(w);
            for (uint32_t i = lane; i < count; i += 32) f(pts[i], level, colorId);
        }
        if (numItems <= numWarps) break;
        uint32_t nx = 0;
        if (lane == 0) nx = atomicAdd(head, 1u);
        it = numWarps + __shfl_sync(0xffffffffu, nx, 0);
    }
}

// The same walk for passes whose per-sample work is "compute a pixel, look at it, maybe update it" with one pixel per
// sample (pointSize 1): ILP samples of a lane are in flight together — their 16-byte loads first, then their framebuffer
// probes — instead of one dependent load chain per sample. A small frame has fewer items than warps, so its draw time IS
// that chain: 1000 samples / 32 lanes = 32 trips of (sample load + probe) per warp.
#ifndef SIMLOD_DRAW_ILP
#define SIMLOD_DRAW_ILP 8              // tuning knob (tools/render_times.py --flags)
#endif
template <typename Prep, typename Probe, typename Commit>
__device__ __forceinline__ void forEachSampleStaged(const uint8_t* heapBase, const WorkItem* items, uint32_t numItems, uint32_t* head,
                                                    Prep&& prep, Probe&& probe, Commit&& commit) {
    constexpr int ILP = SIMLOD_DRAW_ILP;
    const uint32_t lane = laneId();
    const uint32_t numWarps = (gridDim.x * blockDim.x) >> 5;
    uint32_t it = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;
    while (it < numItems) {
        WorkItem w = items[it];
        if (w != ITEM_EMPTY && w != 0) {
            const uint4* pts = itemSamples(heapBase, w);
            const uint32_t count = itemCount(w), level = itemLevel(w), colorId = itemColorId(w);
            for (uint32_t i0 = lane; i0 < count; i0 += 32 * ILP) {
                uint4 p[ILP];
                uint32_t pixel[ILP];
                uint64_t value[ILP], seen[ILP];
#pragma unroll
                for (int u = 0; u < ILP; u++) { const uint32_t i = i0 + 32u * u; p[u] = i < count ? pts[i] : make_uint4(0, 0, 0, 0); }
#pragma unroll
                for (int u = 0; u < ILP; u++) { pixel[u] = 0xffffffffu; value[u] = 0; if (i0 + 32u * u < count) prep(p[u], level, colorId, pixel[u], value[u]); }
#pragma unroll
                for (int u = 0; u < ILP; u++) seen[u] = pixel[u] != 0xffffffffu ? probe(pixel[u]) : 0ull;
#pragma unroll
                for (int u = 0; u < ILP; u++) if (pixel[u] != 0xffffffffu) commit(pixel[u], value[u], seen[u]);
            }
        }
        if (numItems <= numWarps) break;
        uint32_t nx = 0;
        if (lane == 0) nx = atomicAdd(head, 1u);
        it = numWarps + __shfl_sync(0xffffffffu, nx, 0);
    }
}

// ------------------------------------------------------------------------------------------
// bounding-box overlay (Uniforms::showBoundingBox): the 8 edges of the visibility frustum in blue and the 12 edges of
// every drawn node's box in green, as 1-pixel lines (reference render.cu:1195-1227,637-688, rasterization.cuh:5-47,90-183,
// math.cuh:22-152). The reference appends 8 + 48 lines per drawn node to a list and rasterises it one thread per line;
// here line l of [0, 8 + 12 |D|) is derived from its index (its 4 boxes per node are the same box: s = 1 exactly), and a
// warp walks one line, its lanes taking every 32nd step. The frame is a set of 64-bit atomicMins, so neither order nor
// duplicates change it.
// ------------------------------------------------------------------------------------------
constexpr uint32_t OVERLAY_FRUSTUM_LINES = 8, OVERLAY_BOX_LINES = 12;
constexpr uint32_t OVERLAY_FRUSTUM_COLOR = 0x000000ffu, OVERLAY_BOX_COLOR = 0x0000ff00u;

// what the overlay reads of the uniforms, staged in shared memory by the kernel (a kernel parameter cannot be passed by
// reference into a function that is not inlined without a local copy of it), and the clip planes it derives
struct OverlayShared {
    Row T[4];                 // transform: clipping and projection
    Row Tinv[4];              // transformInv_updateBound: the frustum's corners
    float cmin[3], cmax[3], cubeSize;       // boxMin, boxMax, and cubeSizeOf() of them
    float plane[6][4];        // Frustum::fromWorldViewProj(transform): normal, constant
};

// plane p of the frustum of T, rows[3] -+ rows[0..2], normalised (math.cuh:55-64,66-106): boxInFrustum's planes of another
// matrix
__device__ __forceinline__ void overlayPlane(const Row* T, int p, float* out) {
    const Row& a = T[3];
    const Row& b = T[p == 0 || p == 1 ? 0 : (p == 2 || p == 3 ? 1 : 2)];
    const bool minus = (p == 0 || p == 3 || p == 4);
    const float px = minus ? fpx::sub(a.x, b.x) : fpx::add(a.x, b.x);
    const float py = minus ? fpx::sub(a.y, b.y) : fpx::add(a.y, b.y);
    const float pz = minus ? fpx::sub(a.z, b.z) : fpx::add(a.z, b.z);
    const float pw = minus ? fpx::sub(a.w, b.w) : fpx::add(a.w, b.w);
    const float inv = fpx::rcp(fpx::sqrt_approx(dot3(px, py, pz, px, py, pz)));
    out[0] = fpx::mul_ftz(px, inv); out[1] = fpx::mul_ftz(py, inv); out[2] = fpx::mul_ftz(pz, inv); out[3] = fpx::mul_ftz(pw, inv);
}

// Frustum::contains (math.cuh:139-150): dot(n, p) + c < 0 compiles to c < -dot(n, p)
__device__ __forceinline__ bool overlayContains(const OverlayShared& s, float x, float y, float z) {
    bool in = true;
#pragma unroll
    for (int p = 0; p < 6; p++) {
        const float* q = s.plane[p];
        if (q[3] < -dot3(q[0], q[1], q[2], x, y, z)) in = false;
    }
    return in;
}

// Frustum::intersectRay (math.cuh:108-137) with distanceToPlane (math.cuh:28-53): origin + dir * the farthest finite positive
// plane distance, -Infinity when there is none
__device__ __forceinline__ void overlayClip(const OverlayShared& s, float& x, float& y, float& z, float dx, float dy, float dz) {
    const float INF = __int_as_float(0x7f800000);
    float farthest = -INF;
#pragma unroll
    for (int p = 0; p < 6; p++) {
        const float* q = s.plane[p];
        const float den = dot3(q[0], q[1], q[2], dx, dy, dz);
        float d = INF;
        if (den >= 0.0f) {
            const float v = fpx::add(q[3], dot3(q[0], q[1], q[2], x, y, z));
            if (den != 0.0f) { const float t = fpx::mul_ftz(v, -fpx::rcp(den)); if (t >= 0.0f) d = t; }
            else if (v == 0.0f) d = 0.0f;
        }
        if (d > 0.0f && d != INF) farthest = fpx::max_ftz(farthest, d);
    }
    x = fpx::fma(dx, farthest, x); y = fpx::fma(dy, farthest, y); z = fpx::fma(dz, farthest, z);
}

// endpoints of overlay line l (start -> end, as the reference appends them)
__device__ __forceinline__ uint32_t overlayLine(const OverlayShared& s, const Node* nodes, const uint32_t* visList, uint32_t l, float* a, float* b) {
    if (l < OVERLAY_FRUSTUM_LINES) {
        // render.cu:1201-1222: NDC corners through transformInv_updateBound; x, y of start and end, z = -1 -> fend (edges 0-3)
        // or fend -> fend (4-7)
        constexpr float fend = 0.99995f;
        // bit l set: coordinate +1 of line l, else -1 (x, y of the start, then of the end)
        constexpr uint32_t SX = 0x83u, SY = 0x25u, EX = 0xb3u, EY = 0xe5u;
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const float cx = (((k == 0 ? SX : EX) >> l) & 1u) ? 1.0f : -1.0f;
            const float cy = (((k == 0 ? SY : EY) >> l) & 1u) ? 1.0f : -1.0f;
            const float cz = (k == 0 && l < 4) ? -1.0f : fend;
            const float rw = fpx::rcp(rowDot(s.Tinv[3], cx, cy, cz));
            float* o = k == 0 ? a : b;
            o[0] = fpx::mul_ftz(rowDot(s.Tinv[0], cx, cy, cz), rw);
            o[1] = fpx::mul_ftz(rowDot(s.Tinv[1], cx, cy, cz), rw);
            o[2] = fpx::mul_ftz(rowDot(s.Tinv[2], cx, cy, cz), rw);
        }
        return OVERLAY_FRUSTUM_COLOR;
    }
    // drawNodesBoundingBoxes (render.cu:646-687) and drawBoundingBox (rasterization.cuh:25-47): centre
    // cubeMin + float(X + 0.5f) * scale, corners centre -+ scale / 2.0, as its SASS computes them
    const uint32_t v = (l - OVERLAY_FRUSTUM_LINES) / OVERLAY_BOX_LINES, e = (l - OVERLAY_FRUSTUM_LINES) % OVERLAY_BOX_LINES;
    const Node* node = &nodes[visList[v]];
    const float scale = fpx::mul_ftz(s.cubeSize, fpx::ex2(-fpx::u2f(node->level)));
    const float half = fpx::mul_ftz(scale, 0.5f);
    const uint32_t X[3] = {node->X, node->Y, node->Z};
    float mn[3], mx[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float c = fpx::fma(scale, fpx::add(fpx::u2f(X[i]), 0.5f), s.cmin[i]);
        mn[i] = fpx::add(c, -half); mx[i] = fpx::add(c, half);
    }
    // corners as bits x = 4, y = 2, z = 1: the bottom square, the top square, then the four vertical edges
    // (octal digit e, from the right: start corners 0 4 6 2 1 5 7 3 4 6 2 0, end corners 4 6 2 0 5 7 3 1 5 7 3 1)
    constexpr uint64_t FROM = 026437512640ull, TO = 0137513750264ull;
    const uint32_t cf = (uint32_t)(FROM >> (3 * e)) & 7u, ct = (uint32_t)(TO >> (3 * e)) & 7u;
    a[0] = (cf & 4) ? mx[0] : mn[0]; a[1] = (cf & 2) ? mx[1] : mn[1]; a[2] = (cf & 1) ? mx[2] : mn[2];
    b[0] = (ct & 4) ? mx[0] : mn[0]; b[1] = (ct & 2) ? mx[1] : mn[1]; b[2] = (ct & 1) ? mx[2] : mn[2];
    return OVERLAY_BOX_COLOR;
}

// rasterizeLines for one line, by a whole warp (rasterization.cuh:90-183)
__device__ __forceinline__ void overlayRasterLine(const OverlayShared& s, uint64_t* framebuffer, int width, int height,
                                                  float* a, float* b, uint32_t color) {
    const uint32_t lane = laneId();
    float dx = fpx::sub(b[0], a[0]), dy = fpx::sub(b[1], a[1]), dz = fpx::sub(b[2], a[2]);
    const float r = fpx::rsqrt(dot3(dx, dy, dz, dx, dy, dz));               // normalize(): v * rsqrt(dot(v, v))
    dx = fpx::mul(dx, r); dy = fpx::mul(dy, r); dz = fpx::mul(dz, r);
    if (!overlayContains(s, a[0], a[1], a[2])) overlayClip(s, a[0], a[1], a[2], dx, dy, dz);
    if (!overlayContains(s, b[0], b[1], b[2])) overlayClip(s, b[0], b[1], b[2], -dx, -dy, -dz);

    const Row* T = s.T;
    const float ws = rowDot(T[3], a[0], a[1], a[2]), rs = fpx::rcp(ws);
    const float xs = fpx::mul_ftz(rowDot(T[0], a[0], a[1], a[2]), rs), ys = fpx::mul_ftz(rowDot(T[1], a[0], a[1], a[2]), rs);
    const float we = rowDot(T[3], b[0], b[1], b[2]), re = fpx::rcp(we);
    const float xe = fpx::mul_ftz(rowDot(T[0], b[0], b[1], b[2]), re), ye = fpx::mul_ftz(rowDot(T[1], b[0], b[1], b[2]), re);
    const float fw = (float)width, fh = (float)height;
    const double dw = (double)width, dh = (double)height;
    // length(screen_end - screen_start): the difference contracted into an FFMA, z = 1 - 1 adding a +0
    const float sdx = fpx::fma(fw, fpx::fma(xe, 0.5f, 0.5f), -fpx::mul(fw, fpx::fma(xs, 0.5f, 0.5f)));
    const float sdy = fpx::fma(fh, fpx::fma(ye, 0.5f, 0.5f), -fpx::mul(fh, fpx::fma(ys, 0.5f, 0.5f)));
    const float len = fpx::sqrt_approx(fpx::add(0.0f, fpx::fma(sdx, sdx, fpx::mul(sdy, sdy))));
    const float steps = fpx::max_ftz(0.0f, fpx::min_ftz(len, 400.0f));       // clamp(steps, 0, 400): a NaN length gives 400
    const float stepSize = fpx::rcp_rn(steps);                                 // float(1.0 / steps)
    const double xs64 = fpx::f2d(xs), ys64 = fpx::f2d(ys), ws64 = fpx::f2d(ws);

    // for (u = 0; u <= 1.0; u += stepSize): the float recurrence is serial, so every lane runs all of it and draws the
    // steps k0 + lane; stepSize > 0, so the steps drawn are a prefix
    float u = 0.0f;
    for (;;) {
        float mine = 0.0f;
#pragma unroll
        for (uint32_t j = 0; j < 32; j++) { if (j == lane) mine = u; u = fpx::add(stepSize, u); }
        if (mine <= 1.0f) {
            const double omu = fpx::dadd(1.0, -fpx::f2d(mine));
            const float nx = fpx::d2f(fpx::dfma(xs64, omu, fpx::f2d(fpx::mul(xe, mine))));
            const float ny = fpx::d2f(fpx::dfma(ys64, omu, fpx::f2d(fpx::mul(ye, mine))));
            if (!(nx < -1.0f || nx > 1.0f || ny < -1.0f || ny > 1.0f)) {
                const float depth = fpx::d2f(fpx::dfma(ws64, omu, fpx::f2d(fpx::mul(we, mine))));
                int x = fpx::d2i(fpx::dmul(dw, fpx::dfma(fpx::f2d(nx), 0.5, 0.5)));
                int y = fpx::d2i(fpx::dmul(dh, fpx::dfma(fpx::f2d(ny), 0.5, 0.5)));
                x = max(min(x, width - 1), 0); y = max(min(y, height - 1), 0);
                uint64_t* px = &framebuffer[(uint32_t)(x + width * y)];
                const uint64_t value = ((uint64_t)__float_as_uint(depth) << 32) | color;
                if (value < *px) atomicMin(reinterpret_cast<unsigned long long*>(px), (unsigned long long)value);
            }
        }
        if (!(u <= 1.0f)) break;
    }
}

// the end of a frame (render.cu:1244-1343): Stats, then eye-dome lighting and the RGBA8 surface
__device__ __forceinline__ void finishFrame(RCtl* ctl, Stats* stats, uint32_t frameID, uint64_t* framebuffer, cudaSurfaceObject_t gl_colorbuffer,
                                            int width, int height, uint32_t numPixels, bool first, uint32_t gtid, uint32_t gstride) {
    if (first) {      // render.cu:1244-1252
        stats->numVisibleNodes = ldv(&ctl->cutCount);
        ctl->cutCount = 0; ctl->cutMagic = CUT_MAGIC;           // for the next frame (nothing reads the counter after the items phase)
        stats->numVisibleInner = ldv(&ctl->numVisibleInner);
        stats->numVisibleLeaves = ldv(&ctl->numVisibleLeaves);
        stats->numVisiblePoints = ldv(&ctl->numVisiblePoints);
        stats->numVisibleVoxels = ldv(&ctl->numVisibleVoxels);
        stats->frameID = frameID;
    }

    // eye-dome lighting over 16x16 tiles (render.cu:1255-1325). Always on; covers
    // floor(numTiles / gridDim.x) * gridDim.x tiles (sic: the remainder keeps its raw colour).
    {
        struct Pixel { uint32_t color; float depth; };
        Pixel* fbp = reinterpret_cast<Pixel*>(framebuffer);
        const uint32_t tileSize = 16;
        const uint32_t numTilesX = (uint32_t)width / tileSize, numTilesY = (uint32_t)height / tileSize;
        const uint32_t numTiles = numTilesX * numTilesY;
        const uint32_t tilesPerBlock = numTiles / gridDim.x;
#ifndef SIMLOD_EDL_SYNC
#define SIMLOD_EDL_SYNC 1              // tuning knob: the reference's two block barriers per tile (nothing here needs them)
#endif
        for (uint32_t i = 0; i < tilesPerBlock; i++) {
            if (SIMLOD_EDL_SYNC) __syncthreads();
            int tileID = (int)(i * gridDim.x + blockIdx.x);
            int tileX = tileID % (int)numTilesX, tileY = tileID / (int)numTilesX;
            int tileStart = tileX * (int)tileSize + tileY * width * (int)tileSize;
            int pixelID = tileStart + (int)(threadIdx.x % tileSize) + (int)(threadIdx.x / tileSize) * width;
            Pixel pixel = fbp[pixelID];
            float lp = fpx::lg2(pixel.depth);
            float sum = 0.0f;
            const int offs[4] = {width, 1, -width, -1};           // int(1.5*sin(u)) + width*int(1.5*cos(u)), u = 0, PI/2, PI, 3PI/2
#pragma unroll
            for (int k = 0; k < 4; k++) {
                int index = pixelID + offs[k];
                index = max(index, 0);
                index = min(index, width * height);
                float nd = fbp[index].depth;
                double diff = (double)fpx::add(lp, -fpx::lg2(nd));
                sum = (float)fpx::dadd((double)sum, fmax(diff, 0.0));
            }
            float response = fpx::mul_ftz(sum, 0.02f);                         // sum / numSamples(50)
            float e = (float)fpx::dmul(fpx::dmul((double)response, 300.0), (double)0.4f);
            float shade = fpx::ex2(fpx::mul(e, -1.4426950216293334961f));     // __expf(-response * 300.0 * edlStrength)
            uint32_t R = fpx::f2u(fpx::mul(shade, (float)(pixel.color & 0xffu)));
            uint32_t G = fpx::f2u(fpx::mul(shade, (float)((pixel.color >> 8) & 0xffu)));
            uint32_t B = fpx::f2u(fpx::mul(shade, (float)((pixel.color >> 16) & 0xffu)));
            const uint32_t shaded = R | (G << 8) | (B << 16) | 0xff000000u;
            fbp[pixelID].color = shaded;
            // colour -> RGBA8 surface (render.cu:1334-1343), fused: EDL only ever reads neighbours' depths
            surf2Dwrite(shaded, gl_colorbuffer, (pixelID % width) * 4, pixelID / width);
            if (SIMLOD_EDL_SYNC) __syncthreads();
        }
        // pixels outside the tiles the EDL pass covers keep their raw colour
        const uint32_t tilesCovered = tilesPerBlock * gridDim.x;
        for (uint32_t i = gtid; i < numPixels; i += gstride) {
            const uint32_t x = i % (uint32_t)width, y = i / (uint32_t)width;
            const uint32_t tx = x / tileSize, ty = y / tileSize;
            const bool covered = tx < numTilesX && ty < numTilesY && ty * numTilesX + tx < tilesCovered;
            if (!covered) surf2Dwrite((uint32_t)(framebuffer[i] & 0xffffffffull), gl_colorbuffer, (int)x * 4, (int)y);
        }
    }
}

__shared__ OverlayShared overlayShared;

// A frame with the overlay, from the end of the draw on, by every thread of the grid: the lines, one warp per line, then
// the rest of the frame. The kernel has filled in the uniforms of overlayShared; thread 0..5 of the block add the planes.
__device__ __noinline__ void overlayFrame(uint8_t* base, Stats* stats, uint32_t frameID, const Node* nodes,
                                          cudaSurfaceObject_t gl_colorbuffer, int width, int height) {
    RCtl* ctl = reinterpret_cast<RCtl*>(base + rbuf::OFF_CTL);
    const uint32_t* visList = reinterpret_cast<const uint32_t*>(base + rbuf::OFF_VISLIST);
    uint64_t* framebuffer = reinterpret_cast<uint64_t*>(base + rbuf::OFF_FB);
    OverlayShared& s = overlayShared;
    __syncthreads();
    if (threadIdx.x < 6) overlayPlane(s.T, threadIdx.x, s.plane[threadIdx.x]);
    if (threadIdx.x == 6)      // cubeSizeOf
        s.cubeSize = fmaxf(fmaxf(fpx::sub(s.cmax[0], s.cmin[0]), fpx::sub(s.cmax[1], s.cmin[1])), fpx::sub(s.cmax[2], s.cmin[2]));
    __syncthreads();
    const uint32_t numDrawn = min(ldv(&ctl->cutCount), (uint32_t)rbuf::VIS_CAP);
    const uint32_t numLines = OVERLAY_FRUSTUM_LINES + OVERLAY_BOX_LINES * numDrawn;
    const uint32_t numWarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t l = (threadIdx.x >> 5) * gridDim.x + blockIdx.x; l < numLines; l += numWarps) {
        float a[3], b[3];
        const uint32_t color = overlayLine(s, nodes, visList, l, a, b);
        overlayRasterLine(s, framebuffer, width, height, a, b, color);
    }
    cg::grid_group grid = cg::this_grid();
    grid.sync();
    finishFrame(ctl, stats, frameID, framebuffer, gl_colorbuffer, width, height, (uint32_t)(width * height), grid.thread_rank() == 0,
                blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}

// ------------------------------------------------------------------------------------------
// kernel_render, and simlod_render_clip: the same frame with the samples a clip volume excludes left out (DESIGN.md §9.15).
// simlod_render_clip takes kernel_render's arguments and the clip by value, so the clip lives in the kernel-parameter
// constant bank. It is launched on kernel_render's grid, which the EDL tile coverage depends on, with a mode of INSIDE or
// OUTSIDE: without a clip the host launches kernel_render.
// ------------------------------------------------------------------------------------------
extern "C" __global__ void __launch_bounds__(256, 4)
kernel_render(uint32_t* buffer, const Uniforms uniforms, Node* nodes, cudaSurfaceObject_t gl_colorbuffer,
              Stats* stats, uint64_t* frameStartTimestamp, CudaPrint* cudaprint) {
#define SIMLOD_DRAW_CLIP(p)
#include "render_frame.inc"
#undef SIMLOD_DRAW_CLIP
}

extern "C" __global__ void __launch_bounds__(256, 4)
simlod_render_clip(uint32_t* buffer, const Uniforms uniforms, Node* nodes, cudaSurfaceObject_t gl_colorbuffer,
                   Stats* stats, uint64_t* frameStartTimestamp, CudaPrint* cudaprint, const SimlodClip clip) {
#define SIMLOD_DRAW_CLIP(p) if (!clipKeeps(clip, __uint_as_float(p.x), __uint_as_float(p.y), __uint_as_float(p.z))) return;
#include "render_frame.inc"
#undef SIMLOD_DRAW_CLIP
}
