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

namespace cg = cooperative_groups;

typedef SimlodPoint Point;
typedef SimlodChunk Chunk;
typedef SimlodNode Node;
typedef SimlodStats Stats;
typedef SimlodUniforms Uniforms;
typedef SimlodFloat4 Row;
struct CudaPrint;

// render-buffer layout. The framebuffer and the HQS targets sit where the reference's bump
// allocator puts them (render.cu:1108-1123,172,224-231), so both kernels can be read back with
// the same offsets; the area the reference uses for 100 000 Node copies holds our work queue, and the
// unused tail of the 200 000 000-byte buffer (main.cpp:556) a cache of the nodes' chunk lists.
namespace rbuf {
constexpr uint64_t OFF_CTL       = 0;
constexpr uint64_t OFF_VISLIST   = 4096;                           // u32 node indices of the LOD cut
constexpr uint64_t VIS_CAP       = 263168;
constexpr uint64_t ITEM_CAP      = 2097152;                        // chunk items per frame = 2 G samples (the reference: 100 000 nodes)
constexpr uint64_t OFF_ITEMS     = OFF_VISLIST + VIS_CAP * 4;      // u64 per item, see packItem()
constexpr uint64_t OFF_FB        = 31200144;                       // 15 200 000 + 7*16 + 32 + 16 000 000
constexpr uint64_t TOTAL_BYTES   = 200000000;                      // what the host allocates (main.cpp:556)
constexpr uint64_t NODE_TAB      = 263168;                         // >= floor(40 000 000 / 152) nodes
static_assert(OFF_ITEMS + ITEM_CAP * 8 <= OFF_FB, "render scratch overlaps the framebuffer");
}

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

__constant__ uint32_t SPECTRAL[8] = {0x4f3ed5, 0x436df4, 0x61aefd, 0x8be0fe, 0x98f5e6, 0xa4ddab, 0xa5c266, 0xbd8832};

__device__ __forceinline__ uint32_t ldv(const uint32_t* p) { return *(volatile const uint32_t*)p; }
__device__ __forceinline__ uint32_t laneId() { return threadIdx.x & 31; }
__device__ __forceinline__ uint64_t globaltimer() { uint64_t t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

// mat4 row * (x, y, z, 1): y*r.y -> fma(x, r.x) -> fma(z, r.z) -> + r.w   (helper_math.h:1266 as contracted in the reference SASS)
__device__ __forceinline__ float rowDot(const Row& r, float x, float y, float z) {
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
__device__ __forceinline__ bool boxIsLarge(const Uniforms& u, const NodeBox& bx) {
    const Row* T = u.transform_updateBound.rows;
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
__device__ __forceinline__ bool boxInFrustum(const Uniforms& u, const NodeBox& bx) {
    const Row* T = u.transform_updateBound.rows;
    bool inFrustum = true;
#pragma unroll
    for (int p = 0; p < 6 && inFrustum; p++) {
        const Row& a = T[3];
        const Row& b = T[p == 0 || p == 1 ? 0 : (p == 2 || p == 3 ? 1 : 2)];
        bool minus = (p == 0 || p == 3 || p == 4);
        float px = minus ? fpx::sub(a.x, b.x) : fpx::add(a.x, b.x);
        float py = minus ? fpx::sub(a.y, b.y) : fpx::add(a.y, b.y);
        float pz = minus ? fpx::sub(a.z, b.z) : fpx::add(a.z, b.z);
        float pw = minus ? fpx::sub(a.w, b.w) : fpx::add(a.w, b.w);
        if (planeRejects(px, py, pz, pw, bx.mn[0], bx.mn[1], bx.mn[2], bx.mx[0], bx.mx[1], bx.mx[2])) inFrustum = false;
    }
    return inFrustum;
}

__device__ __forceinline__ bool isLeaf(const Node* node) {
    bool leaf = true;
#pragma unroll
    for (int i = 0; i < 8; i++) leaf = leaf && node->children[i] == nullptr;
    return leaf;
}

// One thread per node: the node's flags (render.cu:762-901) and, in the same phase, the LOD cut (render.cu:906-933). A
// node is drawn when it is a visible non-large child of a large node, or a large visible leaf. The parent's `isLarge` is a
// function of the parent's coordinates (level - 1, X/2, Y/2, Z/2) and the frozen update transform alone, so the child
// recomputes it instead of waiting for the thread that owns the parent: no barrier between the flags and the cut.
__device__ void computeVisibilityAndCut(const Uniforms& u, Node* nodes, uint32_t numNodes, float cubeSize,
                                        float cminx, float cminy, float cminz, RCtl* ctl, uint32_t* visList) {
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < numNodes; n += stride) {
        Node* node = &nodes[n];
        const uint32_t level = node->level, X = node->X, Y = node->Y, Z = node->Z;
        const NodeBox bx = nodeBox(level, X, Y, Z, cubeSize, cminx, cminy, cminz);
        const bool large = boxIsLarge(u, bx);
        const bool hasSamples = node->numPoints > 0 || node->numVoxels > 0;
        const bool visible = hasSamples && boxInFrustum(u, bx);
        node->visible = visible ? 1 : 0;
        node->isLarge = large ? 1 : 0;
        if (!visible) continue;
        bool drawn;
        if (large) drawn = isLeaf(node);
        else drawn = level > 0 && boxIsLarge(u, nodeBox(level - 1, X >> 1, Y >> 1, Z >> 1, cubeSize, cminx, cminy, cminz));
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

// Node::getID() % 127 (structures.cuh:116-143, render.cu:74-76), with its arithmetic as compiled: the first nine digits
// are shifted as 32-bit ints (wrap, then sign-extend into the 64-bit id), the rest as 64-bit values; unused name bytes
// are 0, i.e. digit -48
__device__ __forceinline__ uint32_t nodeColorId(const Node* node) {
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
// projection of one sample (render.cu:61-70)
// ------------------------------------------------------------------------------------------
struct Projected { int x, y; float depth; bool inside; };

__device__ __forceinline__ Projected project(const Row* T, float width, float height, float px, float py, float pz) {
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

__device__ __forceinline__ uint32_t sampleColor(const Uniforms& u, uint32_t pointColor, uint32_t level, uint32_t colorId) {
    if (u.colorByNode) return (uint32_t)((uint64_t)colorId * 123456789ull);  // (node->getID() % 127) * 123456789 (render.cu:74-76)
    if (u.colorByLOD) {                                                      // render.cu:49-59,76-78
        int index = fpx::f2i(fpx::mul((float)(8 - (int)level), 1.8f));
        index = max(0, min(index, 7));
        return SPECTRAL[index];
    }
    return pointColor;
}

// ------------------------------------------------------------------------------------------
// kernel_render
// ------------------------------------------------------------------------------------------
extern "C" __global__ void __launch_bounds__(256, 4)
kernel_render(uint32_t* buffer, const Uniforms uniforms, Node* nodes, cudaSurfaceObject_t gl_colorbuffer,
              Stats* stats, uint64_t* frameStartTimestamp, CudaPrint* cudaprint) {
    cg::grid_group grid = cg::this_grid();
    const bool first = grid.thread_rank() == 0;
    const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t gstride = gridDim.x * blockDim.x;

    uint8_t* base = reinterpret_cast<uint8_t*>(buffer);
    RCtl* ctl = reinterpret_cast<RCtl*>(base + rbuf::OFF_CTL);
    WorkItem* items = reinterpret_cast<WorkItem*>(base + rbuf::OFF_ITEMS);
    uint64_t* framebuffer = reinterpret_cast<uint64_t*>(base + rbuf::OFF_FB);

    const int width = fpx::f2i(uniforms.width), height = fpx::f2i(uniforms.height);
    const uint32_t numPixels = (uint32_t)(width * height);
    // HQS targets follow the framebuffer (render.cu:172,224-231: 4-byte counter rounded to 16, depth, colour)
    const uint64_t fbBytes = (uint64_t)numPixels * 8;
    uint32_t* fb_depth = reinterpret_cast<uint32_t*>(base + rbuf::OFF_FB + ((fbBytes + 15) & ~15ull) + 16);
    uint32_t* fb_color = fb_depth + (((uint64_t)numPixels * 4 + 15) & ~15ull) / 4;
    const bool hqs = uniforms.useHighQualityShading != 0;

    // chunk-list cache: whatever the 200 000 000-byte buffer has left behind the HQS targets
    EmitCtx ec;
    ec.ctl = ctl; ec.items = items; ec.nodes = nodes;
    {
        const uint64_t cacheOff = ((uint64_t)(reinterpret_cast<uint8_t*>(fb_color + 4ull * numPixels) - base) + 255ull) & ~255ull;
        const uint64_t entriesBytes = rbuf::NODE_TAB * 2 * sizeof(ListEntry);
        ec.cache = reinterpret_cast<CacheHeader*>(base + cacheOff);
        ec.entries = reinterpret_cast<ListEntry*>(base + cacheOff + 256);
        ec.pool = reinterpret_cast<uint64_t*>(base + cacheOff + 256 + entriesBytes);
        const uint64_t poolOff = cacheOff + 256 + entriesBytes;
        ec.poolCap = poolOff + (1ull << 20) <= rbuf::TOTAL_BYTES ? (uint32_t)min((rbuf::TOTAL_BYTES - poolOff) / 8, (uint64_t)0x7fffffffu) : 0u;
    }
    // the persistent heap: the root's grid is its first allocation, right behind the 16-byte header {buffer, offset}
    // (reset.cu:40-43,69 of the reference and ours)
    ec.heapBase = reinterpret_cast<const uint8_t*>(nodes[0].grid) - 16;
    ec.heapUsed = nodes[0].grid ? *reinterpret_cast<const volatile uint64_t*>(ec.heapBase + 8) : 0ull;

    const bool cutCounterReady = ctl->cutMagic == CUT_MAGIC;      // (see RCtl)
    // developer timers (tools/render_times.py builds a -DSIMLOD_RENDER_TIMERS=1 variant): off in the shipped build, every warp
    // pays for the `first` test at each site
#ifndef SIMLOD_RENDER_TIMERS
#define SIMLOD_RENDER_TIMERS 0
#endif
    uint64_t tPhase = globaltimer();
#if SIMLOD_RENDER_TIMERS
#define RPHASE(k) do { if (first) { uint64_t _t = globaltimer(); ctl->phaseNanos[k] = _t - tPhase; tPhase = _t; } } while (0)
#else
#define RPHASE(k) do { } while (0)
#endif
    if (first) {
        *frameStartTimestamp = tPhase;
        ctl->numItems = 0; ctl->head[0] = 0; ctl->head[1] = 0; ctl->head[2] = 0;
        ctl->numVisiblePoints = 0; ctl->numVisibleVoxels = 0;
        if (!cutCounterReady) ctl->cutCount = 0;
        ctl->numVisibleInner = 0; ctl->numVisibleLeaves = 0; ctl->overflow = 0;
        ctl->cacheHits = 0; ctl->cacheWalks = 0;
        if (ec.poolCap != 0 && (ec.cache->magic != CACHE_MAGIC || ec.cache->poolCap != ec.poolCap || ec.cache->cursor >= ec.poolCap)) {
            // first frame, another resolution, another kernel's scratch, or the pool ran full: start the pool over (stale
            // entries are harmless: they fail verification)
            ec.cache->magic = CACHE_MAGIC; ec.cache->cursor = 0; ec.cache->poolCap = ec.poolCap;
        }
    }
    if (!cutCounterReady) grid.sync();
    // ---- phase 1: clear the targets | visibility flags of every node + LOD cut (independent) ----------------------
    // clear: depth = +inf (0x7f800000), colour = 0x00332211 (render.cu:1126-1131)
    {
        const uint64_t clearValue = (0x7f800000ull << 32) | 0x00332211ull;
        ulonglong2* fb2 = reinterpret_cast<ulonglong2*>(framebuffer);
        for (uint32_t i = gtid; i < numPixels / 2; i += gstride) fb2[i] = make_ulonglong2(clearValue, clearValue);
        if ((numPixels & 1) && first) framebuffer[numPixels - 1] = clearValue;
        if (hqs && uniforms.showPoints) {
            for (uint32_t i = gtid; i < numPixels; i += gstride) fb_depth[i] = 0x7f800000u;
            uint4* c4 = reinterpret_cast<uint4*>(fb_color);
            for (uint32_t i = gtid; i < numPixels; i += gstride) c4[i] = make_uint4(0, 0, 0, 0);
        }
    }
    float bsx = fpx::sub(uniforms.boxMax[0], uniforms.boxMin[0]);
    float bsy = fpx::sub(uniforms.boxMax[1], uniforms.boxMin[1]);
    float bsz = fpx::sub(uniforms.boxMax[2], uniforms.boxMin[2]);
    float cubeSize = fmaxf(fmaxf(bsx, bsy), bsz);
    const uint32_t numNodes = min(ldv(&stats->numNodes), (uint32_t)rbuf::NODE_TAB);
    uint32_t* visList = reinterpret_cast<uint32_t*>(base + rbuf::OFF_VISLIST);
    computeVisibilityAndCut(uniforms, nodes, numNodes, cubeSize, uniforms.boxMin[0], uniforms.boxMin[1], uniforms.boxMin[2], ctl, visList);
    grid.sync();
    RPHASE(0);
    RPHASE(1);

    // ---- phase 2: chunk items of the drawn nodes ------------------------------------------------------------------
    if (nodes[0].grid != nullptr) emitVisible(ec, visList, min(ldv(&ctl->cutCount), (uint32_t)rbuf::VIS_CAP));
    grid.sync();
    RPHASE(2);

    const uint32_t numItems = min(ldv(&ctl->numItems), (uint32_t)rbuf::ITEM_CAP);
    const Row* T = uniforms.transform.rows;
    const int pointSize = uniforms.pointSize;
    const uint8_t* heapBase = ec.heapBase;

    if (uniforms.showPoints && !hqs && pointSize == 1) {
        // single pass, one pixel per sample: depth|colour packed in 64 bits, atomicMin (render.cu:61-104,161-210)
        forEachSampleStaged(heapBase, items, numItems, &ctl->head[0],
            [&](uint4 p, uint32_t level, uint32_t colorId, uint32_t& pixel, uint64_t& value) {
                Projected pr = project(T, uniforms.width, uniforms.height, __uint_as_float(p.x), __uint_as_float(p.y), __uint_as_float(p.z));
                if (!pr.inside) return;
                value = ((uint64_t)__float_as_uint(pr.depth) << 32) | sampleColor(uniforms, p.w, level, colorId);
                uint32_t qx = (uint32_t)max(0, min(pr.x, width)), qy = (uint32_t)max(0, min(pr.y, height));      // (render.cu:91-92)
                pixel = qx + (uint32_t)width * qy;
            },
            [&](uint32_t pixel) { return framebuffer[pixel]; },
            [&](uint32_t pixel, uint64_t value, uint64_t seen) {
                if (value < seen) atomicMin(reinterpret_cast<unsigned long long*>(&framebuffer[pixel]), (unsigned long long)value);
            });
    } else if (uniforms.showPoints && !hqs) {
        // single pass: depth|colour packed in 64 bits, atomicMin (render.cu:61-104,161-210)
        forEachSample(heapBase, items, numItems, &ctl->head[0], [&](uint4 p, uint32_t level, uint32_t colorId) {
            Projected pr = project(T, uniforms.width, uniforms.height, __uint_as_float(p.x), __uint_as_float(p.y), __uint_as_float(p.z));
            if (!pr.inside) return;
            uint64_t encoded = ((uint64_t)__float_as_uint(pr.depth) << 32) | sampleColor(uniforms, p.w, level, colorId);
            for (int ox = 0; ox < pointSize; ox++)
            for (int oy = 0; oy < pointSize; oy++) {
                uint32_t qx = (uint32_t)max(0, min(pr.x + ox, width));        // clamp bounds are inclusive (render.cu:91-92)
                uint32_t qy = (uint32_t)max(0, min(pr.y + oy, height));
                uint32_t pixelID = qx + (uint32_t)width * qy;
                if (encoded < framebuffer[pixelID]) atomicMin(reinterpret_cast<unsigned long long*>(&framebuffer[pixelID]), (unsigned long long)encoded);
            }
        });
    } else if (uniforms.showPoints && hqs && pointSize == 1) {
        // the two HQS passes with one pixel per sample, staged like the single pass above
        auto prepHqs = [&](uint4 p, uint32_t level, uint32_t colorId, uint32_t& pixel, uint64_t& value) {
            Projected pr = project(T, uniforms.width, uniforms.height, __uint_as_float(p.x), __uint_as_float(p.y), __uint_as_float(p.z));
            if (!pr.inside || !(pr.depth > 0.0f)) return;
            value = ((uint64_t)__float_as_uint(pr.depth) << 32) | sampleColor(uniforms, p.w, level, colorId);
            uint32_t qx = (uint32_t)max(0, min(pr.x, width)), qy = (uint32_t)max(0, min(pr.y, height));
            pixel = qx + (uint32_t)width * qy;
        };
        auto probeDepth = [&](uint32_t pixel) { return (uint64_t)fb_depth[pixel]; };
        // pass 1: closest depth per pixel (render.cu:247-391)
        forEachSampleStaged(heapBase, items, numItems, &ctl->head[1], prepHqs, probeDepth,
            [&](uint32_t pixel, uint64_t value, uint64_t seen) {
                const uint32_t udepth = (uint32_t)(value >> 32);
                if (udepth < (uint32_t)seen) atomicMin(&fb_depth[pixel], udepth);
            });
        grid.sync();
        // pass 2: accumulate colours of samples within 1 % of the closest depth (render.cu:406-602)
        forEachSampleStaged(heapBase, items, numItems, &ctl->head[2], prepHqs, probeDepth,
            [&](uint32_t pixel, uint64_t value, uint64_t seen) {
                const float depth = __uint_as_float((uint32_t)(value >> 32)), fbDepth = __uint_as_float((uint32_t)seen);
                const uint32_t color = (uint32_t)value;
                if (depth < fpx::mul(fbDepth, 1.01f)) {
                    // the four 32-bit sums {R, G, B, n} of render.cu:560-580 as two 64-bit adds on the same 16 bytes: a low half
                    // cannot carry into the high one (255 x samples per pixel < 2^32)
                    unsigned long long* acc = reinterpret_cast<unsigned long long*>(&fb_color[4 * pixel]);
                    atomicAdd(acc + 0, (unsigned long long)(color & 0xffu) | ((unsigned long long)((color >> 8) & 0xffu) << 32));
                    atomicAdd(acc + 1, (unsigned long long)((color >> 16) & 0xffu) | (1ull << 32));
                }
            });
        grid.sync();
    } else if (uniforms.showPoints && hqs) {
        // pass 1: closest depth per pixel (render.cu:247-391)
        forEachSample(heapBase, items, numItems, &ctl->head[1], [&](uint4 p, uint32_t level, uint32_t colorId) {
            Projected pr = project(T, uniforms.width, uniforms.height, __uint_as_float(p.x), __uint_as_float(p.y), __uint_as_float(p.z));
            if (!pr.inside || !(pr.depth > 0.0f)) return;
            uint32_t udepth = __float_as_uint(pr.depth);
            for (int ox = 0; ox < pointSize; ox++)
            for (int oy = 0; oy < pointSize; oy++) {
                uint32_t qx = (uint32_t)max(0, min(pr.x + ox, width));
                uint32_t qy = (uint32_t)max(0, min(pr.y + oy, height));
                uint32_t pixelID = qx + (uint32_t)width * qy;
                if (udepth < fb_depth[pixelID]) atomicMin(&fb_depth[pixelID], udepth);
            }
        });
        grid.sync();
        // pass 2: accumulate colours of samples within 1 % of the closest depth (render.cu:406-602)
        forEachSample(heapBase, items, numItems, &ctl->head[2], [&](uint4 p, uint32_t level, uint32_t colorId) {
            Projected pr = project(T, uniforms.width, uniforms.height, __uint_as_float(p.x), __uint_as_float(p.y), __uint_as_float(p.z));
            if (!pr.inside || !(pr.depth > 0.0f)) return;
            uint32_t color = sampleColor(uniforms, p.w, level, colorId);
            for (int ox = 0; ox < pointSize; ox++)
            for (int oy = 0; oy < pointSize; oy++) {
                uint32_t qx = (uint32_t)max(0, min(pr.x + ox, width));
                uint32_t qy = (uint32_t)max(0, min(pr.y + oy, height));
                uint32_t pixelID = qx + (uint32_t)width * qy;
                float fbDepth = __uint_as_float(fb_depth[pixelID]);
                if (pr.depth < fpx::mul(fbDepth, 1.01f)) {
                    atomicAdd(&fb_color[4 * pixelID + 0], color & 0xffu);
                    atomicAdd(&fb_color[4 * pixelID + 1], (color >> 8) & 0xffu);
                    atomicAdd(&fb_color[4 * pixelID + 2], (color >> 16) & 0xffu);
                    atomicAdd(&fb_color[4 * pixelID + 3], 1u);
                }
            }
        });
        grid.sync();
    }
    if (uniforms.showPoints && hqs) {
        // resolve (render.cu:606-632)
        for (uint32_t i = gtid; i < numPixels; i += gstride) {
            uint4 acc = reinterpret_cast<const uint4*>(fb_color)[i];
            if (acc.w == 0) continue;
            uint32_t color = ((acc.x / acc.w) & 0xffu) | (((acc.y / acc.w) & 0xffu) << 8) | (((acc.z / acc.w) & 0xffu) << 16) | 0xff000000u;
            framebuffer[i] = ((uint64_t)fb_depth[i] << 32) | color;
        }
    }
    grid.sync();
    RPHASE(3);

    // the line/bounding-box overlay of the reference (render.cu:1197-1233) is empty unless
    // showBoundingBox is set; it is a debug overlay and not part of this path.

    if (first) {      // render.cu:1244-1252
        stats->numVisibleNodes = ldv(&ctl->cutCount);
        ctl->cutCount = 0; ctl->cutMagic = CUT_MAGIC;           // for the next frame (nothing reads the counter after the items phase)
        stats->numVisibleInner = ldv(&ctl->numVisibleInner);
        stats->numVisibleLeaves = ldv(&ctl->numVisibleLeaves);
        stats->numVisiblePoints = ldv(&ctl->numVisiblePoints);
        stats->numVisibleVoxels = ldv(&ctl->numVisibleVoxels);
        stats->frameID = (uint32_t)uniforms.frameCounter;
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
    RPHASE(4);
}
