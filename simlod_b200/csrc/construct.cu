// construct.cu — incremental octree/LOD builder for sm_90a (H100).
//
// Drop-in for the reference's `kernel_construct`
// (modules/progressive_octree/progressive_octree_voxels.cu:804-1010): same extern "C"
// name, same argument list, same Node/Chunk/OccupancyGrid/Stats contents afterwards
// (canonical form: DESIGN.md §3), launched cooperatively with 256-thread blocks by
// updateOctree() (main_progressive_octree.cpp:364-428). It is NOT a translation of that
// kernel; what is preserved is the observable state, what is new is how it is computed:
//
//   reference                                           here
//   ------------------------------------------------    ------------------------------------------
//   3 full passes over the batch (count, voxel-         1 streaming pass (count + voxel-sample fused),
//   sample, insert), each re-descending the tree        leaf id + slot cached per point (8 B), 1 insert pass
//   via 64-byte children[] pointer arrays               descent through a 4 B/node first-child table,
//                                                       skipped when the point falls into the thread's last leaf
//   voxel sampling top-down, one bitmap probe per       bottom-up from the deepest inner node, stops at the first
//   level of the path (voxels.cu:426-470)               set bit: occupancy bits are nested across levels
//   contiguous-per-thread ranges (uncoalesced)          TMA-staged contiguous block runs, 128-bit shared loads
//   atomicAdd(numPoints) per point at insert            slot = block-aggregated counter add (no atomics at insert)
//   chunk lists walked i/1000 hops per point/voxel      chunk rows / per-batch chunk directory: O(1) address
//   one thread walks/extends each node's list           tail pointers kept per node; only dirty nodes visited
//   1 global atomic per created voxel (backlog)         block-local ranks, one add per node per block
//   >= 24 grid-wide barriers per batch                  1 (+2 per split round): allocation and insertion of
//                                                       batch b-1 run inside the counting phase of batch b
//
// The scratch ("momentary") buffer is carved with our own layout (namespace scratch); it fits in
// the 300 000 000 bytes the unmodified host allocates (main_progressive_octree.cpp:554),
// unlike the reference's carve-out which needs 408 800 192 (voxels.cu:834-856).
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
typedef SimlodHeapHeader Heap;
struct CudaPrint;   // opaque: the reference's debug channel is a dead parameter (CudaPrint.cuh:51)

// ------------------------------------------------------------------------------------------
// scratch layout inside the momentary buffer (all offsets 256-byte aligned). Everything that the
// insertion of batch b-1 reads while batch b is being counted exists twice (index = batch parity).
// ------------------------------------------------------------------------------------------
namespace scratch {
constexpr uint64_t NODE_CAP       = 263157;            // floor(40 000 000 / 152): the nodes the host allocates (main.cpp:552-555)
constexpr uint64_t NODE_TAB       = 263168;            // side-table length (NODE_CAP rounded up)
constexpr uint64_t MAX_BATCH      = SIMLOD_MAX_BATCH_SIZE;
constexpr uint64_t SPILL_CAP      = 3ull << 20;        // spilled points per batch (the reference re-inserts <= 3 000 001, voxels.cu:628)
constexpr uint64_t ITEM_CAP       = MAX_BATCH + SPILL_CAP;
constexpr uint64_t VOXEL_CAP      = 4ull << 20;        // voxels created per batch, per parity
constexpr uint64_t VOXEL_SHARED   = 512ull << 10;      // tail of the voxel backlog shared by all blocks (overflow of a block's own segment)
constexpr uint64_t DIR_CAP        = 512ull << 10;      // chunk directory entries per batch, per parity
constexpr uint64_t QUEUE_CAP      = 3ull << 19;        // free-chunk stack, 1.5 Mi entries (reference: 1 M)
constexpr uint64_t WL_CAP         = 2ull << 20;        // items a re-walk round can be told to visit by name (more: every affected run is scanned)
constexpr uint64_t SPILLNODE_CAP  = 100000;            // voxels.cu:847
constexpr uint64_t ROW_CAP        = 65536;             // leaves that hold points at the same time (x 64 chunk slots)
constexpr uint64_t ROW_SLOTS      = 64;                // chunk pointers per leaf row (a leaf holds <= 50 chunks)
constexpr uint64_t BLOCK_CAP      = 4096;              // per-block cursor slots (grid sizes up to 4096 blocks)

constexpr uint64_t align256(uint64_t x) { return (x + 255) & ~255ull; }
constexpr uint64_t OFF_CTL        = 0;
constexpr uint64_t OFF_FIRSTCHILD = 4096;
constexpr uint64_t OFF_PARENT     = align256(OFF_FIRSTCHILD + NODE_TAB * 4);
constexpr uint64_t OFF_GRIDPTR    = align256(OFF_PARENT + NODE_TAB * 4);
constexpr uint64_t OFF_LEAFROW    = align256(OFF_GRIDPTR + NODE_TAB * 8);
constexpr uint64_t OFF_SPLITSTATE = align256(OFF_LEAFROW + NODE_TAB * 4);
constexpr uint64_t OFF_VTAIL      = align256(OFF_SPLITSTATE + NODE_TAB * 4);
constexpr uint64_t OFF_VDIR       = align256(OFF_VTAIL + NODE_TAB * 8);
constexpr uint64_t OFF_DIRTYLEAF  = align256(OFF_VDIR + NODE_TAB * 8);                 // [2]
constexpr uint64_t OFF_DIRTYVOX   = align256(OFF_DIRTYLEAF + 2 * NODE_TAB * 4);        // [2]
constexpr uint64_t OFF_SPILLINFO  = align256(OFF_DIRTYVOX + 2 * NODE_TAB * 4);
constexpr uint64_t OFF_BLOCKCUR   = align256(OFF_SPILLINFO + SPILLNODE_CAP * 32);      // [2]
constexpr uint64_t OFF_RUNBLOOM   = align256(OFF_BLOCKCUR + 2 * BLOCK_CAP * 4);          // [BLOCK_CAP][8]
constexpr uint64_t OFF_RUNFLAG    = align256(OFF_RUNBLOOM + BLOCK_CAP * 32);             // [BLOCK_CAP]
constexpr uint64_t OFF_ROWFREE    = align256(OFF_RUNFLAG + BLOCK_CAP * 4);
constexpr uint64_t OFF_ROWS       = align256(OFF_ROWFREE + ROW_CAP * 4);
constexpr uint64_t OFF_CHUNKDIR   = align256(OFF_ROWS + ROW_CAP * ROW_SLOTS * 8);      // [2]
constexpr uint64_t OFF_QUEUE      = align256(OFF_CHUNKDIR + 2 * DIR_CAP * 8);
constexpr uint64_t OFF_LEAFOF     = align256(OFF_QUEUE + QUEUE_CAP * 8);               // [2]
constexpr uint64_t OFF_SLOTOF     = align256(OFF_LEAFOF + 2 * ITEM_CAP * 4);           // [2]
constexpr uint64_t OFF_SPILLED    = align256(OFF_SLOTOF + 2 * ITEM_CAP * 4);
constexpr uint64_t OFF_VKEY       = align256(OFF_SPILLED + SPILL_CAP * 16);            // [2]
constexpr uint64_t OFF_VCOLOR     = align256(OFF_VKEY + 2 * VOXEL_CAP * 8);            // [2]
constexpr uint64_t OFF_WORKLIST   = align256(OFF_VCOLOR + 2 * VOXEL_CAP * 4);
constexpr uint64_t TOTAL          = align256(OFF_WORKLIST + WL_CAP * 4);
static_assert(TOTAL <= 300000000ull, "scratch must fit the host's 300 MB momentary buffer (main.cpp:554)");
}  // namespace scratch

enum : uint32_t {   // Ctl::errorFlags, mirrored into Stats::dbg. Sticky: cleared only by a reset (batchletIndex == 0).
    ERR_SPILL_OVERFLOW  = 1u << 0,   // more than SPILL_CAP spilled points in one batch: a split was postponed (reference-undefined regime)
    ERR_VOXEL_OVERFLOW  = 1u << 1,   // more than VOXEL_CAP voxels created in one batch: voxels were dropped
    ERR_DIR_OVERFLOW    = 1u << 2,
    ERR_NODE_OVERFLOW   = 1u << 3,   // nodes[] capacity exceeded: a split was refused
    ERR_QUEUE_OVERFLOW  = 1u << 4,
    ERR_SPILLNODE_OVERFLOW = 1u << 5,
    ERR_ROW_OVERFLOW    = 1u << 6,   // more than ROW_CAP non-empty leaves, or a leaf with more than 64 chunks: points were dropped
    ERR_FAR_POINT       = 1u << 7,   // a point further than 16 cube edges outside the box (its 2^28 and 2^20 quantisations disagree)
    ERR_INTERNAL        = 1u << 8,   // an invariant of the builder itself was violated (never seen; reported rather than ignored)
};

struct BatchCounters {              // one set per batch, index = batch % 3; the idle set is cleared during the phase before its use
    uint32_t numSpillTotal;        // spilling nodes found so far in this batch (monotonic)
    uint32_t numSpilled;           // spilled points in this batch
    uint32_t numBacklog;           // voxels of this batch that went to the shared overflow part of the backlog
    uint32_t numDirtyLeaves;
    uint32_t numDirtyVox;
    uint32_t dirCursor;
    uint32_t voxelsCreated;        // voxels of this batch (bound for the capacity guard)
    uint32_t insertCursor;         // next tile of the batch's insertion work to hand out
};

struct Ctl {
    uint32_t numBatchesUploaded;   // snapshot of the volatile host-updated counter (voxels.cu:872-876)
    uint32_t errorFlags;
    uint64_t elapsedNanos;
    uint64_t memUsed;              // heap offset snapshot for the capacity guard
    uint32_t rowBump;              // leaf rows handed out so far (persistent across launches)
    uint32_t rowFreeCount;         // entries on the row free stack (persistent)
    uint32_t statCounters[8];      // @32
    uint64_t voxelsByPass[2];      // @64 voxels created in first-visit passes / in re-walk passes since the last reset
    uint64_t spilledTotal;         // @80 spilled (re-inserted) points since the last reset: the `s` of the roofline's 32*s bytes
    uint64_t voxelsTotal;          // @88 voxels created since the last reset (incl. leaf-root voxels)
    uint64_t phaseNanos[8];        // @96 time per phase since reset, by the grid's first thread (%globaltimer):
                                   //     0 fused phase (alloc b-1 | count+sample b | insert b-1), 1 split round, 2 re-walk, 3 deferred sampling,
                                   //     4 final allocate, 5 final insert + stats, 6 split rounds run, 7 launch prologue
    BatchCounters batch[3];        // @160
    uint32_t allocDone;            // @256 blocks that have finished their share of the in-phase allocations of this launch (monotonic)
    uint32_t _pad[3];
    uint64_t launchClock[32][2];   // %globaltimer at the start / end of the last 32 launches (slot = launchCount % 32): launch gaps as the device sees them
    uint32_t launchCount, _pad2[3];
    uint64_t subNanos[16];         // @800
                                   //      block 0's own timeline inside the phases (developer aid): fused = 0 allocate, 1 count+sample, 2 wait for the
                                   //      allocation, 3 flush, 4 insert, 5 barrier; split = 6 work, 7 barrier; re-walk = 8 items, 9 flush, 10 barrier;
                                   //      11 top of the batch loop, 12-14 re-walk set-up / listed items / spilled points
    struct Worklist { uint32_t cursor[2]; uint32_t legacy; uint32_t pad; } wl[3];      // @928 per batch (index = batch % 3): entries of the list of
                                   //      round r (cursor[r & 1]); legacy != 0: some block could not name its items, rounds scan the affected runs
    uint32_t events[4];            // @976 since the last reset: re-walk rounds run in legacy mode, warps that counted globally for lack of list room,
                                   //      table-full global counts, splits refused
    uint64_t elapsedByParity[2];   // @992 launch time at the end of the fused phase of the last even / odd batch (read by the snapshots of that batch)
    uint64_t roundHist[12][4];     // @1008 timers build: re-walk rounds by size class (class = bit length of listed + spilled items, / 2, capped):
                                   //       rounds, nanoseconds (split + re-walk), listed items, spilled items of the round
};
static_assert(offsetof(Ctl, roundHist) == 1008 && sizeof(Ctl) <= 4096, "tools read Ctl by offset; the control block is 4 KB");
static_assert(offsetof(Ctl, events) == 976, "tools read Ctl by offset");
static_assert(offsetof(Ctl, spilledTotal) == 80, "bench.py reads Ctl::spilledTotal at byte 80");
static_assert(offsetof(Ctl, phaseNanos) == 96 && offsetof(Ctl, batch) == 160 && offsetof(Ctl, allocDone) == 256 && offsetof(Ctl, launchClock) == 272 && offsetof(Ctl, launchCount) == 784 && offsetof(Ctl, subNanos) == 800, "tools read Ctl by offset");

// what the lane that sees a leaf cross 50 000 records about it (everything the split round needs)
struct SpillInfo {
    uint32_t node;
    uint32_t stored;       // points the leaf held before this batch
    uint32_t base;         // where they go in the spill buffer
    uint32_t row;          // the leaf's chunk row (+1)
    uint32_t childBase;    // index of child 0
    uint32_t level;
    uint64_t grid;         // occupancy grid of the new inner node
};
static_assert(sizeof(SpillInfo) == 32, "SpillInfo");

struct DirEntry { uint32_t base; uint32_t k0; };   // chunkDir[base + (slot/1000 - k0)] holds element `slot`

// Everything is addressed from the kernel's own parameters (constant bank) plus compile-time
// offsets, so the context is a handful of registers and never lives in local memory.
struct Ctx {
    uint8_t*   buf;           // momentary buffer
    Node*      nodes;
    Stats*     stats;
    uint8_t*   heapBytes;
    float minx, miny, minz, size, rcpSize;
    uint32_t   segCap;        // backlog entries per block segment

    template <typename T> __device__ __forceinline__ T* at(uint64_t off) const { return reinterpret_cast<T*>(buf + off); }
    __device__ __forceinline__ Heap*      heap()        const { return reinterpret_cast<Heap*>(heapBytes); }
    __device__ __forceinline__ Ctl*       ctl()         const { return at<Ctl>(scratch::OFF_CTL); }
    __device__ __forceinline__ uint32_t*  firstChild()  const { return at<uint32_t>(scratch::OFF_FIRSTCHILD); }   // node -> index of child 0 (8 consecutive nodes); 0 = leaf
    __device__ __forceinline__ uint32_t*  parentOf()    const { return at<uint32_t>(scratch::OFF_PARENT); }
    __device__ __forceinline__ uint64_t*  gridPtr()     const { return at<uint64_t>(scratch::OFF_GRIDPTR); }      // node -> OccupancyGrid* (0 = none)
    __device__ __forceinline__ uint32_t*  leafRow()     const { return at<uint32_t>(scratch::OFF_LEAFROW); }      // leaf -> row of its chunk pointers (+1; 0 = none)
    __device__ __forceinline__ uint32_t*  splitState()  const { return at<uint32_t>(scratch::OFF_SPLITSTATE); }   // leaf -> 1 once its split has been requested
    __device__ __forceinline__ uint64_t*  voxelTail()   const { return at<uint64_t>(scratch::OFF_VTAIL); }        // node -> last Chunk* of its voxel list
    __device__ __forceinline__ DirEntry*  voxelDir()    const { return at<DirEntry>(scratch::OFF_VDIR); }
    __device__ __forceinline__ uint32_t*  dirtyLeaves(uint32_t p) const { return at<uint32_t>(scratch::OFF_DIRTYLEAF) + p * scratch::NODE_TAB; }
    __device__ __forceinline__ uint32_t*  dirtyVox(uint32_t p)    const { return at<uint32_t>(scratch::OFF_DIRTYVOX) + p * scratch::NODE_TAB; }
    __device__ __forceinline__ SpillInfo* spill()       const { return at<SpillInfo>(scratch::OFF_SPILLINFO); }
    __device__ __forceinline__ uint32_t*  blockCursor(uint32_t p) const { return at<uint32_t>(scratch::OFF_BLOCKCUR) + p * scratch::BLOCK_CAP; }
    __device__ __forceinline__ uint32_t*  runBloom()    const { return at<uint32_t>(scratch::OFF_RUNBLOOM); }     // [block][8]: leaves the block's run of the batch sits in
    __device__ __forceinline__ uint32_t*  runFlag()     const { return at<uint32_t>(scratch::OFF_RUNFLAG); }      // [block]: the run must be revisited in the coming re-walk pass
    __device__ __forceinline__ uint32_t*  rowFree()     const { return at<uint32_t>(scratch::OFF_ROWFREE); }
    __device__ __forceinline__ uint64_t*  rows()        const { return at<uint64_t>(scratch::OFF_ROWS); }         // [ROW_CAP][64] chunk pointers of leaves, in list order
    __device__ __forceinline__ uint64_t*  chunkDir(uint32_t p) const { return at<uint64_t>(scratch::OFF_CHUNKDIR) + p * scratch::DIR_CAP; }
    __device__ __forceinline__ uint64_t*  chunkQueue()  const { return at<uint64_t>(scratch::OFF_QUEUE); }
    __device__ __forceinline__ uint32_t*  leafOf(uint32_t p) const { return at<uint32_t>(scratch::OFF_LEAFOF) + p * scratch::ITEM_CAP; }   // item -> leaf node | level << 24
    __device__ __forceinline__ uint32_t*  slotOf(uint32_t p) const { return at<uint32_t>(scratch::OFF_SLOTOF) + p * scratch::ITEM_CAP; }   // item -> index inside the leaf
    __device__ __forceinline__ Point*     spilled()     const { return at<Point>(scratch::OFF_SPILLED); }
    __device__ __forceinline__ uint64_t*  vkey(uint32_t p)   const { return at<uint64_t>(scratch::OFF_VKEY) + p * scratch::VOXEL_CAP; }     // cell | node << 21 | slot << 41
    __device__ __forceinline__ uint32_t*  vcolor(uint32_t p) const { return at<uint32_t>(scratch::OFF_VCOLOR) + p * scratch::VOXEL_CAP; }
    __device__ __forceinline__ uint32_t*  worklist()    const { return at<uint32_t>(scratch::OFF_WORKLIST); }    // items (leafOf index) the coming re-walk pass visits
};

// the batch a pass works on
struct Batch {
    const Point* points;     // ring slot
    uint32_t size;
    uint32_t index;          // global batch index (Stats::batchletIndex of this batch)
    uint32_t parity;         // index & 1: which copy of the per-batch arrays
    BatchCounters* bc;       // &ctl->batch[index % 3]
};

// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------
// values other blocks wrote in an earlier phase (or that the host's copies wrote): read at the L2, never from a stale L1 line.
// (ld.relaxed.gpu rather than a volatile load: the latter is a system-scope access, several times the latency)
__device__ __forceinline__ uint32_t ldv(const uint32_t* p) { uint32_t v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ uint64_t ldv(const uint64_t* p) { uint64_t v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ uint32_t ldcg(const uint32_t* p) { uint32_t v; asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p)); return v; }
__device__ __forceinline__ uint32_t ldAcquire(const uint32_t* p) { uint32_t v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ uint32_t laneId() { return threadIdx.x & 31; }
__device__ __forceinline__ bool first_in_grid() { return blockIdx.x == 0 && threadIdx.x == 0; }
__device__ __forceinline__ uint32_t lanemaskLt() { uint32_t m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
__device__ __forceinline__ uint64_t globaltimer() { uint64_t t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

__device__ __forceinline__ uint4 ldPoint(const Point* p) {     // streaming 128-bit load
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void stPoint(Point* p, uint4 v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

struct Coords { uint32_t X, Y, Z, pX, pY, pZ; };

// voxels.cu:148-155 — X = u32(2^20 * (p - min) / size), pX = u32(2^28 * (p - min) / size)
__device__ __forceinline__ Coords quantize(const Ctx& c, uint4 pt) {
    float dx = fpx::add(__uint_as_float(pt.x), -c.minx);
    float dy = fpx::add(__uint_as_float(pt.y), -c.miny);
    float dz = fpx::add(__uint_as_float(pt.z), -c.minz);
    Coords q;
    q.X  = fpx::f2u(fpx::mul_ftz(fpx::mul(dx, 1048576.0f), c.rcpSize));
    q.Y  = fpx::f2u(fpx::mul_ftz(fpx::mul(dy, 1048576.0f), c.rcpSize));
    q.Z  = fpx::f2u(fpx::mul_ftz(fpx::mul(dz, 1048576.0f), c.rcpSize));
    q.pX = fpx::f2u(fpx::mul_ftz(fpx::mul(dx, 268435456.0f), c.rcpSize));
    q.pY = fpx::f2u(fpx::mul_ftz(fpx::mul(dy, 268435456.0f), c.rcpSize));
    q.pZ = fpx::f2u(fpx::mul_ftz(fpx::mul(dz, 268435456.0f), c.rcpSize));
    return q;
}
// The occupancy cell of level l is bits [21-l, 28-l) of pX, the child taken at level l is bit 19-l of X. For every
// point whose two quantisations agree (X == pX >> 8 on the 20 bits the descent uses: true unless the point lies
// more than 16 cube edges outside the box, where the float -> u32 conversions saturate differently) the cells
// are nested: same node and same level-l cell  =>  same cell in every ancestor's grid.
__device__ __forceinline__ bool nested(const Coords& q) {
    return ((((q.pX >> 8) ^ q.X) | ((q.pY >> 8) ^ q.Y) | ((q.pZ >> 8) ^ q.Z)) & 0xfffffu) == 0;
}
// voxels.cu:171-179
__device__ __forceinline__ uint32_t childIndexAt(const Coords& q, uint32_t level) {
    uint32_t sh = SIMLOD_MAX_DEPTH - 1 - level;
    return (((q.X >> sh) & 1u) << 2) | (((q.Y >> sh) & 1u) << 1) | ((q.Z >> sh) & 1u);
}
// voxels.cu:78-88
__device__ __forceinline__ uint32_t cellAt(const Coords& q, uint32_t level) {
    uint32_t sh = SIMLOD_MAX_DEPTH + 1 - level;
    uint32_t cx = (q.pX >> sh) & 127u, cy = (q.pY >> sh) & 127u, cz = (q.pZ >> sh) & 127u;
    return cx | (cy << 7) | (cz << 14);
}

// ------------------------------------------------------------------------------------------
// The in-phase allocation handshake. Allocation and insertion of batch b-1 run inside the counting
// phase of batch b: every block first allocates its share of b-1's dirty nodes and signals, then
// counts its run of batch b WITHOUT touching anything the allocation reads or writes (leaf counters,
// numPoints, numVoxels[Stored], rows), and only when all blocks have signalled does it flush its
// block-local tables into those fields and insert its share of b-1. All blocks of a cooperative
// launch are co-resident and nobody waits before signalling, so the wait cannot deadlock.
// ------------------------------------------------------------------------------------------
__shared__ uint32_t sh_allocTarget;      // value Ctl::allocDone must reach before this block may touch allocation state (0 = no wait)
__shared__ uint32_t sh_allocSeen;        // set once this block has seen it

__device__ __forceinline__ void waitAllocThread(const Ctx& c) {      // any single thread (slow paths inside the counting loop)
    const uint32_t target = sh_allocTarget;
    if (target == 0 || *(volatile uint32_t*)&sh_allocSeen) return;
    while ((int32_t)(ldAcquire(&c.ctl()->allocDone) - target) < 0) __nanosleep(64);
    *(volatile uint32_t*)&sh_allocSeen = 1;
}
__device__ __forceinline__ void waitAllocBlock(const Ctx& c) {       // whole block, block-uniform
    if (sh_allocTarget != 0) {
        if (threadIdx.x == 0) waitAllocThread(c);
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------
// block-local voxel bookkeeping. A created voxel needs (a) a slot in its node's voxel list =
// numVoxels++ and (b) a backlog entry. For a coherent scan these are two very hot global
// addresses (the upper nodes' counters, the backlog cursor); same-address atomics serialise in L2.
// Instead every block owns a segment of the backlog and a node -> count table in shared memory;
// winners take a block-local rank, and when the block has finished its pass it adds each node's
// count to numVoxels ONCE and patches the entries it wrote with the returned base.
// ------------------------------------------------------------------------------------------
#ifndef SIMLOD_VOXTAB_SIZE
#define SIMLOD_VOXTAB_SIZE 64          // tuning knob (tools/exp_variants.py): power of two, <= 256
#endif
constexpr uint32_t VOXTAB_SIZE = SIMLOD_VOXTAB_SIZE;
static_assert((VOXTAB_SIZE & (VOXTAB_SIZE - 1)) == 0 && VOXTAB_SIZE <= 128, "table size: a power of two, two tables are flushed by one 256-thread block, the index is packed into 7 bits");
constexpr uint32_t VOXTAB_EMPTY = 0xffffffffu;
__shared__ uint32_t sh_tabKey[VOXTAB_SIZE];
__shared__ uint32_t sh_tabCount[VOXTAB_SIZE];
__shared__ uint32_t sh_tabBase[VOXTAB_SIZE];
__shared__ uint32_t sh_cursor;        // next free entry of this block's backlog segment
__shared__ uint32_t sh_passStart;     // first entry written in the current pass

__device__ __forceinline__ uint32_t tabHash(uint32_t key) { return (key * 0x9E3779B1u) >> 26; }
__device__ __forceinline__ uint32_t tabFind(const uint32_t* keys, uint32_t key) {
    uint32_t h = tabHash(key);
#pragma unroll 1
    for (uint32_t probe = 0; probe < VOXTAB_SIZE; probe++) {
        uint32_t s = (h + probe) & (VOXTAB_SIZE - 1);
        uint32_t k = keys[s];
        if (k == key) return s;
        if (k == VOXTAB_EMPTY) break;
    }
    return VOXTAB_EMPTY;
}
__device__ __forceinline__ uint32_t tabInsert(uint32_t* keys, uint32_t key) {
    uint32_t h = tabHash(key);
#pragma unroll 1
    for (uint32_t probe = 0; probe < VOXTAB_SIZE; probe++) {
        uint32_t s = (h + probe) & (VOXTAB_SIZE - 1);
        uint32_t k = atomicCAS(&keys[s], VOXTAB_EMPTY, key);
        if (k == VOXTAB_EMPTY || k == key) return s;
    }
    return VOXTAB_EMPTY;
}

__device__ __forceinline__ void voxelPassBegin(const Ctx& c, const Batch& b, bool firstPassOfBatch) {
    if (threadIdx.x < VOXTAB_SIZE) { sh_tabKey[threadIdx.x] = VOXTAB_EMPTY; sh_tabCount[threadIdx.x] = 0; }
    if (threadIdx.x == 0) { sh_cursor = firstPassOfBatch ? 0u : c.blockCursor(b.parity)[blockIdx.x]; sh_passStart = sh_cursor; }
}

// shared fall-back (block table or block segment full): global atomics, final key at once
__device__ __noinline__ void recordVoxelShared(const Ctx c, const Batch b, uint32_t node, uint32_t cell, uint32_t color) {
    waitAllocThread(c);
    Node* nd = &c.nodes[node];
    uint32_t vslot = atomicAdd(&nd->numVoxels, 1u);
    if (vslot == ldv(&nd->numVoxelsStored)) { uint32_t d = atomicAdd(&b.bc->numDirtyVox, 1u); c.dirtyVox(b.parity)[d] = node; }
    atomicAdd(&b.bc->voxelsCreated, 1u);
    uint32_t e = atomicAdd(&b.bc->numBacklog, 1u);
    if (e < scratch::VOXEL_SHARED) {
        uint64_t at = scratch::VOXEL_CAP - scratch::VOXEL_SHARED + e;
        c.vkey(b.parity)[at] = (uint64_t)cell | ((uint64_t)node << 21) | ((uint64_t)vslot << 41);
        c.vcolor(b.parity)[at] = color;
    } else {
        atomicOr(&c.ctl()->errorFlags, ERR_VOXEL_OVERFLOW);
    }
}

__device__ __forceinline__ void recordVoxel(const Ctx& c, const Batch& b, uint32_t node, uint32_t cell, uint32_t color) {
    // the lanes that arrive here together mostly created their voxel in the same node (a re-walk fills the grid of the
    // node that was just split): one table probe and one add per warp then, instead of one per lane
    const uint32_t active = __activemask();
    const uint32_t leader = __ffs(active) - 1u;
    const uint32_t node0 = __shfl_sync(active, node, leader);
    if (__all_sync(active, node == node0)) {
        const uint32_t n = __popc(active), mine = __popc(active & lanemaskLt());
        uint32_t slot = 0, idx0 = 0, rank0 = 0, fit = 0;      // fit: how many of the n entries still fit the block's segment
        if (laneId() == leader) {
            slot = tabInsert(sh_tabKey, node0);
            if (slot != VOXTAB_EMPTY) {
                idx0 = atomicAdd(&sh_cursor, n);
                fit = idx0 < c.segCap ? min(n, c.segCap - idx0) : 0u;
                if (fit) rank0 = atomicAdd(&sh_tabCount[slot], fit);
            }
        }
        slot = __shfl_sync(active, slot, leader); idx0 = __shfl_sync(active, idx0, leader); rank0 = __shfl_sync(active, rank0, leader); fit = __shfl_sync(active, fit, leader);
        if (mine >= fit) { recordVoxelShared(c, b, node, cell, color); return; }
        const uint64_t at = (uint64_t)blockIdx.x * c.segCap + idx0 + mine;
        c.vkey(b.parity)[at] = (uint64_t)cell | ((uint64_t)slot << 21) | ((uint64_t)(rank0 + mine) << 41);      // node/slot patched in voxelFlushPatch
        c.vcolor(b.parity)[at] = color;
        return;
    }
    uint32_t slot = tabInsert(sh_tabKey, node);
    if (slot == VOXTAB_EMPTY) { recordVoxelShared(c, b, node, cell, color); return; }
    uint32_t idx = atomicAdd(&sh_cursor, 1u);
    if (idx >= c.segCap) { recordVoxelShared(c, b, node, cell, color); return; }
    uint32_t rank = atomicAdd(&sh_tabCount[slot], 1u);
    uint64_t at = (uint64_t)blockIdx.x * c.segCap + idx;
    c.vkey(b.parity)[at] = (uint64_t)cell | ((uint64_t)slot << 21) | ((uint64_t)rank << 41);      // node/slot patched in voxelFlushPatch
    c.vcolor(b.parity)[at] = color;
}

// flush, step 1 (one thread per table entry): add the block's count to the node's numVoxels, remember the base
__device__ __forceinline__ void voxelFlushEntry(const Ctx& c, const Batch& b, uint32_t entry) {
    uint32_t node = sh_tabKey[entry], cnt = sh_tabCount[entry];
    if (node != VOXTAB_EMPTY && cnt > 0) {
        Node* nd = &c.nodes[node];
        uint32_t base = atomicAdd(&nd->numVoxels, cnt);
        if (base == ldv(&nd->numVoxelsStored)) {           // first voxels of this node in this batch
            uint32_t d = atomicAdd(&b.bc->numDirtyVox, 1u);
            c.dirtyVox(b.parity)[d] = node;
        }
        sh_tabBase[entry] = base;
    }
}
// flush, step 2 (whole block, after a barrier): block-local (table slot, rank) -> (node, slot in the node's list)
__device__ __forceinline__ void voxelFlushPatch(const Ctx& c, const Batch& b, bool freshPass) {
    const uint32_t endIdx = min(sh_cursor, c.segCap);
    uint64_t* vkey = c.vkey(b.parity);
    for (uint32_t e = sh_passStart + threadIdx.x; e < endIdx; e += blockDim.x) {
        uint64_t at = (uint64_t)blockIdx.x * c.segCap + e;
        uint64_t k = vkey[at];
        uint32_t slot = (uint32_t)(k >> 21) & (VOXTAB_SIZE - 1);
        uint32_t rank = (uint32_t)(k >> 41);
        vkey[at] = (k & 0x1fffffull) | ((uint64_t)sh_tabKey[slot] << 21) | ((uint64_t)(sh_tabBase[slot] + rank) << 41);
    }
    if (threadIdx.x == 0) {
        c.blockCursor(b.parity)[blockIdx.x] = endIdx;
        if (endIdx > sh_passStart) {
            atomicAdd(&b.bc->voxelsCreated, endIdx - sh_passStart);
            atomicAdd(reinterpret_cast<unsigned long long*>(&c.ctl()->voxelsTotal), (unsigned long long)(endIdx - sh_passStart));
            atomicAdd(reinterpret_cast<unsigned long long*>(&c.ctl()->voxelsByPass[freshPass ? 0 : 1]), (unsigned long long)(endIdx - sh_passStart));
        }
    }
}

// ------------------------------------------------------------------------------------------
// block-local leaf counting. A scan is spatially coherent, so at any moment most of the grid
// counts into the same handful of leaves, and one atomicAdd(counter) per warp per iteration
// (what the reference does, voxels.cu:203-218) makes those counters the hottest addresses of the
// pass — with the returned value on every warp's critical path. Here a warp takes a block-local
// rank from a shared-memory table instead; when the block has finished its pass it adds each
// leaf's total to the global counter once (where the spill / first-touch detection now happens)
// and turns the provisional ranks of its items into slots.
// ------------------------------------------------------------------------------------------
// A provisional slot carries its table entry: bit 31 | entry << 24 | block-local rank (< 2^24: a block never
// counts more than ITEM_CAP items); a final slot (table full, counted globally at once) is the plain index.
constexpr uint32_t PROVISIONAL = 0x80000000u;
static_assert(scratch::ITEM_CAP < (1u << 24), "block-local ranks must fit 24 bits");
__shared__ uint32_t sh_leafKey[VOXTAB_SIZE];
__shared__ uint32_t sh_leafCount[VOXTAB_SIZE];
__shared__ uint32_t sh_leafBase[VOXTAB_SIZE];
__shared__ uint8_t  sh_leafLevel[VOXTAB_SIZE];
__device__ __forceinline__ uint32_t finalSlot(uint32_t sl) { return (sl & PROVISIONAL) ? sh_leafBase[(sl >> 24) & 127u] + (sl & 0xffffffu) : sl; }
// the first-visit pass keeps the slots of the block's own run in shared memory until they are final
constexpr uint32_t RUNSLOT_CAP = 2048;
__shared__ uint32_t sh_runSlot[RUNSLOT_CAP];
// "My items": what the block counted in its last counting pass, with the table entry each went to (the slot word).
// After the first-visit pass that is its run of the batch (sh_runSlot); after a re-walk pass the explicit list below
// (kept in the TMA stages, which only first-visit passes use). A leaf can only cross its capacity in the pass that
// adds to it, so the items that move in a round are exactly items of these lists whose table entry names a leaf that
// was split: the split phase picks them out in shared memory and names them in a global worklist, and the re-walk
// pass visits the worklist — nothing is scanned to find out that it did not move. A block that cannot name its
// items (list or table full, run too long for sh_runSlot) raises Ctl::Worklist::legacy; the rounds of that batch then
// scan the affected runs (markAffectedRun), for which the run filters are kept up to date in every case.
constexpr uint32_t LIST_CAP = 2048;
__shared__ uint32_t sh_listCount;         // entries of the explicit list (may run past LIST_CAP: overflow)
__shared__ uint32_t sh_listMode;          // 0: the run (sh_runSlot), 1: the explicit list
__shared__ uint32_t sh_blockLegacy;       // this block cannot name its items any more in this batch
__shared__ uint8_t  sh_entrySplit[VOXTAB_SIZE];
__shared__ uint32_t sh_splitNodes[64];
__shared__ SpillInfo sh_splitInfo[64];       // the leaves split in the current round (worklist rounds: at most 64) ...
__shared__ uint32_t sh_splitGranule[65];     // ... and the running number of 32-point granules of their spilled points
__shared__ uint32_t sh_wlCount, sh_wlBase, sh_wlFill;
__shared__ uint32_t sh_roundLegacy, sh_roundListed;     // the round's worklist state, loaded once per block after the split barrier
// block-wide exclusive prefix sum of one value per thread (256 threads); returns the block total
__device__ __forceinline__ uint32_t blockExclusiveScan(uint32_t v, uint32_t& total) {
    __shared__ uint32_t sh_warpSum[8];
    __shared__ uint32_t sh_total;
    const uint32_t lane = laneId(), warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += t; }
    __syncthreads();                       // protects sh_* against the previous call
    if (lane == 31) sh_warpSum[warp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t run = 0; for (int w = 0; w < 8; w++) { uint32_t t = sh_warpSum[w]; sh_warpSum[w] = run; run += t; } sh_total = run; }
    __syncthreads();
    total = sh_total;
    return sh_warpSum[warp] + incl - v;
}

// Re-walk rounds visit only the runs of the batch that can hold an item whose leaf was split in the round: every
// run (= the contiguous piece of the batch one block counted in the first-visit pass) keeps a 256-bit Bloom filter of
// the leaves its items sit in — built in shared memory during the first-visit pass, kept in global memory, extended
// when a re-walk moves items of the run into new leaves. A round tests the few leaves it split against all filters,
// and the items of the runs that may be affected are shared out evenly over the WHOLE grid (a false positive costs
// a rescan of that run, never a missed item).
constexpr uint32_t BLOOM_WORDS = 8;
constexpr uint32_t AFFECTED_CAP = 1024;   // grids up to this many blocks build the list; larger ones rescan every run
__shared__ uint32_t sh_runBloom[BLOOM_WORDS];
__shared__ uint32_t sh_affected[AFFECTED_CAP];
__shared__ uint32_t sh_numAffected;
__device__ __forceinline__ uint32_t bloomHash(uint32_t node) { return (node * 0x9E3779B1u) >> 24; }
__device__ __forceinline__ void bloomAdd(uint32_t* bloom, uint32_t node) { uint32_t h = bloomHash(node); atomicOr(&bloom[h >> 5], 1u << (h & 31u)); }

// The items of a re-walk pass, as one index space shared out evenly over the grid:
//   [0, A * perRun)              the affected runs of the batch, concatenated
//   then numSpilled entries      the spilled points of this batch (index MAX_BATCH + j in leafOf / slotOf)
// It is handed out in warp-sized granules, round-robin over ALL warps of the grid (consecutive granules to different
// SMs): a moved item costs a walk and usually a new voxel, an unmoved one a look-up, and both kinds as well as the
// spilled points come in long stretches — every block gets the same mix this way.
struct Rewalk { uint32_t perRun, runItems, total, spilledBefore; bool listed; };
__device__ __forceinline__ Rewalk rewalkSlice(uint32_t numBatch, uint32_t numSpilled, uint32_t spilledBefore) {
    Rewalk r;
    r.perRun = ((numBatch + gridDim.x - 1) / gridDim.x + 31u) & ~31u;
    r.listed = gridDim.x <= AFFECTED_CAP;
    r.runItems = (r.listed ? sh_numAffected : gridDim.x) * r.perRun;
    r.total = r.runItems + numSpilled;
    r.spilledBefore = spilledBefore;
    return r;
}
__device__ __forceinline__ uint32_t rewalkFirstGranule() { return ((threadIdx.x >> 5) * gridDim.x + blockIdx.x) * 32u; }
__device__ __forceinline__ uint32_t rewalkGranuleStride() { return gridDim.x * blockDim.x; }
// index into leafOf / slotOf of item u (0xffffffff: padding of a run); run = the run it belongs to (spilled: none)
__device__ __forceinline__ uint32_t rewalkItem(const Rewalk& r, uint32_t u, uint32_t& run) {
    run = 0xffffffffu;
    if (u >= r.runItems) return (uint32_t)scratch::MAX_BATCH + (u - r.runItems);
    const uint32_t k = u / r.perRun;
    run = r.listed ? sh_affected[k] : k;
    return run * r.perRun + (u - k * r.perRun);
}

// the global step: add `cnt` points to a leaf's counter; first-touch and spill detection (voxels.cu:203-218)
__device__ __noinline__ uint32_t countGlobal(const Ctx c, const Batch b, uint32_t node, uint32_t level, uint32_t cnt) {
    waitAllocThread(c);
    Node* leaf = &c.nodes[node];
    uint32_t old = atomicAdd(&leaf->counter, cnt);
    uint32_t stored = ldv(&leaf->numPoints);
    if (old == stored) {                                     // first points of this leaf in this batch
        uint32_t d = atomicAdd(&b.bc->numDirtyLeaves, 1u);
        c.dirtyLeaves(b.parity)[d] = node;
    }
    // The leaf spills when its counter crosses 50 000 (voxels.cu:211-217). Exactly one adder wins the request; it
    // reserves everything the split needs right here, so the split round is one phase: room in the spill buffer,
    // 8 node slots, the occupancy grid. A split that cannot be served (our capacities, never reached where the
    // reference itself is defined) is refused as a whole and requested again by the next add to that leaf.
    if (old + cnt > SIMLOD_MAX_POINTS_PER_NODE && atomicCAS(&c.splitState()[node], 0u, 1u) == 0u) {
        uint32_t err = 0;
        const uint32_t childBase = atomicAdd(&c.stats->numNodes, 8u);                                // voxels.cu:317
        if ((uint64_t)childBase + 8 > scratch::NODE_CAP) { err = ERR_NODE_OVERFLOW; atomicSub(&c.stats->numNodes, 8u); }
        uint32_t base = 0;
        if (!err && stored) {
            base = atomicAdd(&b.bc->numSpilled, stored);
            if ((uint64_t)base + stored > scratch::SPILL_CAP) { err = ERR_SPILL_OVERFLOW; atomicSub(&b.bc->numSpilled, stored); atomicSub(&c.stats->numNodes, 8u); }
        }
        uint32_t s = 0;
        if (!err) {
            s = atomicAdd(&b.bc->numSpillTotal, 1u);
            if (s >= scratch::SPILLNODE_CAP) {
                err = ERR_SPILLNODE_OVERFLOW; atomicSub(&b.bc->numSpillTotal, 1u);
                if (stored) atomicSub(&b.bc->numSpilled, stored);
                atomicSub(&c.stats->numNodes, 8u);
            }
        }
        if (err) {
            atomicOr(&c.ctl()->errorFlags, err);
            atomicAdd(&c.ctl()->events[3], 1u);
            atomicExch(&c.splitState()[node], 0u);
        } else {
            SpillInfo info;
            info.node = node;
            info.stored = stored;
            info.level = level;
            info.row = c.leafRow()[node];
            info.base = base;
            info.childBase = childBase;
            uint64_t g = c.gridPtr()[node];
            if (g == 0) g = (uint64_t)(c.heapBytes + atomicAdd(reinterpret_cast<unsigned long long*>(&c.heap()->offset), (unsigned long long)SIMLOD_GRID_STRIDE));   // voxels.cu:363-365
            info.grid = g;
            c.spill()[s] = info;
        }
    }
    return old;
}

// ------------------------------------------------------------------------------------------
// the per-point walk. Warp-synchronous: all 32 lanes call it together, `valid` masks lanes
// without an item.
//   descent : voxels.cu:145-187 from (node, level) to the leaf through the first-child table — skipped when
//             the point falls into the leaf this thread found last (a scan is coherent: nearly always)
//   sample  : voxels.cu:426-470 + 50-121. The reference probes the grid of every node on the path, root first.
//             Occupancy bits are nested (see nested()): if the point's cell is set in a node it is set in all its
//             ancestors, or will be before the pass ends by the thread that set it. So the walk goes UP from the
//             deepest inner node and stops at the first set bit: one probe per point plus one per created voxel.
//   count   : voxels.cu:203-218 (doCounting::countPoint)
// ------------------------------------------------------------------------------------------
struct LeafCache { uint32_t node, level, kx, ky, kz, parent; };      // node == VOXTAB_EMPTY: nothing cached

// count (voxels.cu:203-218, doCounting::countPoint): the lanes of a warp that reached the same leaf take consecutive ranks
// from the block's table (or, when the table or the block's item list is full, final slots from the global counter).
// Warp-collective; returns the lane's slot word. `bloom`: the filter of the run the lane's item belongs to (none for
// spilled points). MIXED_RUNS: the lanes' items may come from different runs (the worklist concatenates the blocks'
// segments, so a warp's granule can straddle two of them) — every run gets the leaf, not only the leader's.
template <bool MIXED_RUNS = false>
__device__ __forceinline__ uint32_t countInto(const Ctx& c, const Batch& b, bool valid, uint32_t node, uint32_t level, uint32_t* bloom, bool forceGlobal) {
    const uint32_t lane = laneId();
    uint32_t slot = 0;
    const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
    if (valid) {
        uint32_t peers = __match_any_sync(vmask, node);
        uint32_t leader = __ffs(peers) - 1;
        uint32_t cnt = __popc(peers);
        uint32_t r = 0;
        if (lane == leader) {
            uint32_t t = forceGlobal ? VOXTAB_EMPTY : tabInsert(sh_leafKey, node);
            if (t != VOXTAB_EMPTY) { r = atomicAdd(&sh_leafCount[t], cnt) | PROVISIONAL | (t << 24); sh_leafLevel[t] = (uint8_t)level; }   // block-local rank
            else                 { r = countGlobal(c, b, node, level, cnt); sh_blockLegacy = 1; if (!forceGlobal) atomicAdd(&c.ctl()->events[2], 1u); }   // table (or list) full: final slot at once
            if (bloom) bloomAdd(bloom, node);
        }
        r = __shfl_sync(peers, r, leader);
        slot = r + __popc(peers & lanemaskLt());
        if (MIXED_RUNS) {
            const uint64_t leaderBloom = __shfl_sync(peers, (uint64_t)(uintptr_t)bloom, leader);
            if (bloom && (uint64_t)(uintptr_t)bloom != leaderBloom) bloomAdd(bloom, node);
        }
    }
    return slot;
}

// the upward half of the walk: probe / set the point's cell from (sNode, sLevel) towards the root until a set bit is met
// (or down to stopLevel), recording a voxel for every cell this thread wins
template <bool UNCACHED_GRID, bool DEDUP>
__device__ __forceinline__ void sampleUp(const Ctx& c, const Batch& b, const Coords& q, uint32_t color, uint32_t sNode, uint32_t sLevel, uint32_t stopLevel) {
    const uint32_t lane = laneId();
    const bool exhaustive = !nested(q);          // far outside the box: probe every level like the reference does
    if (exhaustive) atomicOr(&c.ctl()->errorFlags, ERR_FAR_POINT);
    // atomicOr results are not needed to continue upwards (a speculative probe of the level above is always
    // correct: every cell has exactly one winner), so up to 3 stay in flight per lane
    uint32_t pending = 0;
    uint32_t old0 = 0, old1 = 0, old2 = 0, key0 = 0, key1 = 0, key2 = 0, cel0 = 0, cel1 = 0, cel2 = 0;
    auto settle = [&]() {
        if (pending > 0 && (old0 & (1u << (cel0 & 31u))) == 0) recordVoxel(c, b, key0, cel0, color);
        if (pending > 1 && (old1 & (1u << (cel1 & 31u))) == 0) recordVoxel(c, b, key1, cel1, color);
        if (pending > 2 && (old2 & (1u << (cel2 & 31u))) == 0) recordVoxel(c, b, key2, cel2, color);
        pending = 0;
    };
    const uint64_t* gridPtr = c.gridPtr();
    for (;;) {
        uint64_t g = gridPtr[sNode];
        bool goUp = exhaustive;
        if (g != 0) {
            uint32_t cell = cellAt(q, sLevel);
            uint32_t* word = reinterpret_cast<uint32_t*>(g) + (cell >> 5);
            uint32_t bit = 1u << (cell & 31u);
            // non-atomic pre-test (voxels.cu:93-94): bits are only ever set while a grid is live, so a set bit seen
            // through the (non-coherent) L1 is final. The root's grid is cleared in place when the root splits
            // (voxels.cu:370-382): the one pass that follows such a clear reads through L2 instead.
            uint32_t seen = UNCACHED_GRID ? ldcg(word) : *word;
            if ((seen & bit) == 0) {
                // first-visit passes: neighbouring points of a scan hit the same cell, so one atomic per distinct cell
                // among the converged lanes. Re-walk passes fill freshly cleared grids, where the cells of a warp's
                // items are mostly distinct and the match would cost more than the few atomics it saves.
                bool mine = true;
                if (DEDUP) {
                    uint32_t active = __activemask();
                    uint32_t peers = __match_any_sync(active, (uint64_t)(uintptr_t)word * 32ull + (cell & 31u));
                    mine = lane == (uint32_t)__ffs(peers) - 1u;
                }
                if (mine) {
                    if (pending == 3) settle();
                    uint32_t old = atomicOr(word, bit);
                    if (pending == 0) { old0 = old; key0 = sNode; cel0 = cell; }
                    else if (pending == 1) { old1 = old; key1 = sNode; cel1 = cell; }
                    else { old2 = old; key2 = sNode; cel2 = cell; }
                    pending++;
                    goUp = true;
                }
            }
        }
        if (!goUp || sLevel <= stopLevel) break;
        sNode = c.parentOf()[sNode];
        sLevel--;
    }
    settle();
}

template <bool SAMPLE, bool COUNT, bool UNCACHED_GRID, bool DEDUP>
__device__ __forceinline__ void walk(const Ctx& c, const Batch& b, LeafCache& cache, bool valid, uint4 pt, uint32_t node, uint32_t level,
                                     uint32_t stopLevel, uint32_t* bloom, bool forceGlobal, uint32_t& leafPacked, uint32_t& slot) {
    Coords q = quantize(c, pt);
    uint32_t parent = VOXTAB_EMPTY;
    if (valid) {
        const uint32_t mx = q.X & 0xfffffu, my = q.Y & 0xfffffu, mz = q.Z & 0xfffffu;
        const uint32_t csh = SIMLOD_MAX_DEPTH - cache.level;
        if (cache.node != VOXTAB_EMPTY && (mx >> csh) == cache.kx && (my >> csh) == cache.ky && (mz >> csh) == cache.kz) {
            node = cache.node; level = cache.level; parent = cache.parent;
        } else {
            const uint32_t* firstChild = c.firstChild();
            for (;;) {
                if (level >= SIMLOD_MAX_DEPTH) break;                       // voxels.cu:169 loop bound: a level-20 node is the leaf
                uint32_t fc = firstChild[node];
                if (fc == 0) break;
                parent = node;
                node = fc + childIndexAt(q, level);
                level++;
            }
            if (parent == VOXTAB_EMPTY && level > 0) parent = c.parentOf()[node];
            const uint32_t sh = SIMLOD_MAX_DEPTH - level;
            cache.node = node; cache.level = level; cache.parent = parent;
            cache.kx = mx >> sh; cache.ky = my >> sh; cache.kz = mz >> sh;
        }
        if (SAMPLE) {
            // nodes with a grid on the path: the inner nodes, and the root even while it is a leaf (reset.cu:69)
            const uint32_t sNode = level == 0 ? node : parent;
            const uint32_t sLevel = level == 0 ? 0u : level - 1;
            sampleUp<UNCACHED_GRID, DEDUP>(c, b, q, pt.w, sNode, sLevel, stopLevel);
        }
    }
    __syncwarp();

    leafPacked = node | (level << 24);
    if (COUNT) slot = countInto(c, b, valid, node, level, bloom, forceGlobal);
}

// ------------------------------------------------------------------------------------------
// TMA staging of the batch. In a first-visit pass every block streams its contiguous run of the
// batch through two shared-memory stages with 1-D bulk copies (cp.async.bulk ... mbarrier::
// complete_tx, SASS: UBLKCP): one elected thread issues the copy of the next tile while the block
// walks the current one, so the HBM latency of the batch read leaves the critical path and no
// registers or LSU slots are spent on it. Threads then read their point with one LDS.128.
// ------------------------------------------------------------------------------------------
#ifndef SIMLOD_REWALK_L2TEST
#define SIMLOD_REWALK_L2TEST 0         // tuning knob (tools/exp_variants.py): pre-test the freshly cleared grids of a re-walk through L2 instead of L1
#endif
#ifndef SIMLOD_TILE_POINTS
#define SIMLOD_TILE_POINTS 512         // tuning knob: a multiple of 256
#endif
constexpr uint32_t TILE_POINTS = SIMLOD_TILE_POINTS;
static_assert(TILE_POINTS % 256 == 0 && TILE_POINTS >= 256, "a tile is walked in 256-point steps");
__shared__ __align__(128) uint4 sh_tile[2][TILE_POINTS];
__shared__ __align__(8) uint64_t sh_tileBar[2];
__shared__ uint32_t sh_tilePhase[2];       // parity the next wait on each stage has to see (the barriers live for the whole launch)

__device__ __forceinline__ void tileBarInit() {      // once per launch
    if (threadIdx.x == 0) {
        uint32_t b0 = (uint32_t)__cvta_generic_to_shared(&sh_tileBar[0]), b1 = (uint32_t)__cvta_generic_to_shared(&sh_tileBar[1]);
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(b0) : "memory");
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(b1) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        sh_tilePhase[0] = 0; sh_tilePhase[1] = 0;
    }
    __syncthreads();
}
__device__ __forceinline__ void tileLoad(uint32_t stage, const Point* src, uint32_t numPoints) {
    uint32_t bar = (uint32_t)__cvta_generic_to_shared(&sh_tileBar[stage]);
    uint32_t dst = (uint32_t)__cvta_generic_to_shared(&sh_tile[stage][0]);
    uint32_t bytes = numPoints * 16u;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tileWait(uint32_t stage, uint32_t parity) {
    uint32_t bar = (uint32_t)__cvta_generic_to_shared(&sh_tileBar[stage]);
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    } while (!done);
}

// the contiguous run of the batch a block owns in every pass over it
__device__ __forceinline__ void blockRun(uint32_t numBatch, uint32_t& first, uint32_t& end) {
    const uint32_t perBlock = ((numBatch + gridDim.x - 1) / gridDim.x + 31u) & ~31u;
    first = min(numBatch, blockIdx.x * perBlock);
    end = min(numBatch, first + perBlock);
}

// Split phase, every block for its own run: can the run hold an item of one of the leaves split in this round?
// (The filters are only extended during re-walk passes, and the verdicts are read after the barrier that ends the
// split phase, so every block sees the same set of affected runs.)
__device__ __forceinline__ void markAffectedRun(const Ctx& c, const Batch& b, uint32_t spillBegin, uint32_t spillEnd) {
    if (threadIdx.x >= 32) return;
    const uint32_t perRun = ((b.size + gridDim.x - 1) / gridDim.x + 31u) & ~31u;
    uint32_t flag = 0;
    if (blockIdx.x * perRun < b.size) {
        const uint32_t* bloom = c.runBloom() + blockIdx.x * BLOOM_WORDS;
        for (uint32_t k = spillBegin + threadIdx.x; k < spillEnd; k += 32) {
            const uint32_t h = bloomHash(c.spill()[k].node);
            flag |= (ldcg(&bloom[h >> 5]) >> (h & 31u)) & 1u;
        }
        flag = __any_sync(0xffffffffu, flag != 0) ? 1u : 0u;
    }
    if (threadIdx.x == 0) c.runFlag()[blockIdx.x] = flag;
}

// the explicit list lives in the two TMA stages (16 KB): item index and slot word of up to LIST_CAP items
__device__ __forceinline__ uint32_t* listItem() { return reinterpret_cast<uint32_t*>(&sh_tile[0][0]); }
__device__ __forceinline__ uint32_t* listSlot() { return reinterpret_cast<uint32_t*>(&sh_tile[0][0]) + LIST_CAP; }
static_assert(sizeof(sh_tile) >= LIST_CAP * 8, "the explicit item list must fit the TMA stages");

// Split phase, every block: name the items that move in this round (see sh_listCount above) in the global worklist.
__device__ void buildWorklist(const Ctx& c, const Batch& b, uint32_t spillBegin, uint32_t spillEnd, uint32_t round) {
    Ctl::Worklist* w = &c.ctl()->wl[b.index % 3u];
    const uint32_t numSplit = spillEnd - spillBegin;
#ifdef SIMLOD_NO_WORKLIST
    if (true) {                                                         // developer knob: every round scans the affected runs
#else
    if (numSplit > 64u || sh_blockLegacy != 0) {                       // block-uniform
#endif
        if (threadIdx.x == 0) atomicExch(&w->legacy, 1u);
        return;
    }
    uint32_t blockFirst, blockEnd;
    blockRun(b.size, blockFirst, blockEnd);
    const uint32_t mode = sh_listMode;
    const uint32_t total = mode == 0 ? blockEnd - blockFirst : min(sh_listCount, LIST_CAP);
    if (threadIdx.x < numSplit) sh_splitNodes[threadIdx.x] = c.spill()[spillBegin + threadIdx.x].node;
    if (threadIdx.x == 0) { sh_wlCount = 0; sh_wlFill = 0; }
    __syncthreads();
    if (threadIdx.x < VOXTAB_SIZE) {
        const uint32_t key = sh_leafKey[threadIdx.x];
        uint32_t f = 0;
        if (key != VOXTAB_EMPTY) for (uint32_t j = 0; j < numSplit; j++) f |= key == sh_splitNodes[j] ? 1u : 0u;
        sh_entrySplit[threadIdx.x] = (uint8_t)f;
    }
    __syncthreads();
    const uint32_t* words = mode == 0 ? sh_runSlot : listSlot();
    auto movedAt = [&](uint32_t k) { const uint32_t word = words[k]; return (word & PROVISIONAL) != 0 && sh_entrySplit[(word >> 24) & (VOXTAB_SIZE - 1)] != 0; };
    uint32_t cnt = 0;
    for (uint32_t k = threadIdx.x; k < total; k += blockDim.x) cnt += movedAt(k) ? 1u : 0u;
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (laneId() == 0 && cnt) atomicAdd(&sh_wlCount, cnt);
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t n = sh_wlCount;
        uint32_t base = n ? atomicAdd(&w->cursor[round & 1u], n) : 0u;
        if ((uint64_t)base + n > scratch::WL_CAP) { atomicExch(&w->legacy, 1u); base = 0xffffffffu; }
        sh_wlBase = base;
    }
    __syncthreads();
    const uint32_t base = sh_wlBase;
    if (base == 0xffffffffu || sh_wlCount == 0) return;
    uint32_t* wl = c.worklist();
    const uint32_t* items = listItem();
    for (uint32_t k0 = 0; k0 < total; k0 += blockDim.x) {                // block-uniform trip count
        const uint32_t k = k0 + threadIdx.x;
        const bool m = k < total && movedAt(k);
        const uint32_t mask = __ballot_sync(0xffffffffu, m);
        if (mask == 0) continue;
        uint32_t off = 0;
        if (laneId() == 0) off = atomicAdd(&sh_wlFill, (uint32_t)__popc(mask));
        off = __shfl_sync(0xffffffffu, off, 0);
        if (m) wl[base + off + __popc(mask & lanemaskLt())] = mode == 0 ? blockFirst + k : items[k];
    }
}

// ------------------------------------------------------------------------------------------
// one pass over the batch points (ring slot) followed by the spilled points of this batch
//   FRESH  : items start at the root (first visit); otherwise only items whose cached leaf has
//            been split since are walked on, starting at that (now inner) node
//   the table flush (leaf counters, voxel counters) is left to the caller: passFlush()
// ------------------------------------------------------------------------------------------
template <bool SAMPLE, bool COUNT, bool FRESH, bool UNCACHED_GRID>
__device__ __forceinline__ void passItems(const Ctx& c, const Batch& b, uint32_t numSpilled, uint32_t spilledBefore, uint32_t round, uint32_t spillBegin = 0, uint32_t spillEnd = 0) {
    const uint32_t stride = gridDim.x * blockDim.x;
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t* leafOf = c.leafOf(b.parity);
    uint32_t* slotOf = c.slotOf(b.parity);
    uint32_t blockFirst, blockEnd;
    blockRun(b.size, blockFirst, blockEnd);
    LeafCache cache;
    cache.node = VOXTAB_EMPTY; cache.level = 0; cache.kx = cache.ky = cache.kz = 0; cache.parent = VOXTAB_EMPTY;

    if (COUNT && threadIdx.x < VOXTAB_SIZE) { sh_leafKey[threadIdx.x] = VOXTAB_EMPTY; sh_leafCount[threadIdx.x] = 0; }
    if (FRESH && COUNT && threadIdx.x < BLOOM_WORDS) sh_runBloom[threadIdx.x] = 0;
    if (FRESH && COUNT && threadIdx.x == 0) { sh_listMode = 0; sh_listCount = 0; sh_blockLegacy = (blockEnd - blockFirst) > RUNSLOT_CAP ? 1u : 0u; }
    if (SAMPLE) voxelPassBegin(c, b, FRESH);
    __syncthreads();

    if (FRESH) {
        const uint32_t runLen = blockEnd - blockFirst;
        const uint32_t numTiles = (runLen + TILE_POINTS - 1) / TILE_POINTS;
        uint32_t ph0 = sh_tilePhase[0], ph1 = sh_tilePhase[1];
        __syncthreads();
        // (the stages held the explicit item list of the previous batch's rounds: order those generic-proxy writes before the bulk copies)
        if (threadIdx.x == 0) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (threadIdx.x == 0 && numTiles > 0) tileLoad(0, b.points + blockFirst, min(TILE_POINTS, runLen));
        for (uint32_t t = 0; t < numTiles; t++) {
            const uint32_t tileFirst = blockFirst + t * TILE_POINTS;
            if (threadIdx.x == 0 && t + 1 < numTiles)      // stage (t+1)&1 was drained at the barrier that ended iteration t-1
                tileLoad((t + 1) & 1, b.points + tileFirst + TILE_POINTS, min(TILE_POINTS, blockEnd - (tileFirst + TILE_POINTS)));
            if (t & 1) { tileWait(1, ph1); ph1 ^= 1; } else { tileWait(0, ph0); ph0 ^= 1; }
#pragma unroll 1
            for (uint32_t k = 0; k < TILE_POINTS / 256; k++) {
                const uint32_t idx = k * 256 + threadIdx.x;
                const uint32_t i = tileFirst + idx;
                const bool valid = i < blockEnd;
                uint4 pt = valid ? sh_tile[t & 1][idx] : make_uint4(0, 0, 0, 0);
                uint32_t lp = 0, slot = 0;
                walk<SAMPLE, COUNT, UNCACHED_GRID, true>(c, b, cache, valid, pt, 0, 0, 0, COUNT ? sh_runBloom : nullptr, false, lp, slot);
                if (valid && COUNT) {
                    leafOf[i] = lp;
                    if (runLen <= RUNSLOT_CAP) sh_runSlot[i - blockFirst] = slot; else slotOf[i] = slot;
                }
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) { sh_tilePhase[0] = ph0; sh_tilePhase[1] = ph1; }
        if (COUNT && threadIdx.x < BLOOM_WORDS) c.runBloom()[blockIdx.x * BLOOM_WORDS + threadIdx.x] = sh_runBloom[threadIdx.x];
    } else {
        if (sh_roundLegacy == 0) {
            // ---- the items the split phase named (buildWorklist), then the points spilled in this round ---------------------
            const uint32_t numListed = min(sh_roundListed, (uint32_t)scratch::WL_CAP);
            const uint32_t perRun = ((b.size + gridDim.x - 1) / gridDim.x + 31u) & ~31u;
            const uint32_t* wl = c.worklist();
            const uint32_t numSplit = spillEnd - spillBegin;                      // <= 64 in worklist rounds
            if (threadIdx.x < numSplit) sh_splitInfo[threadIdx.x] = c.spill()[spillBegin + threadIdx.x];
            if (threadIdx.x == 0) { sh_listCount = 0; sh_listMode = 1; }          // the list of the previous round has been read (split phase)
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t run = 0;
                for (uint32_t k = 0; k < numSplit; k++) { sh_splitGranule[k] = run; run += (sh_splitInfo[k].stored + 31u) / 32u; }
                sh_splitGranule[numSplit] = run;
            }
            __syncthreads();
#if SIMLOD_TIMERS >= 2
            uint64_t tRw = globaltimer();
#define RW_DONE(k) do { __syncthreads(); if (blockIdx.x == 0 && threadIdx.x == 0) { uint64_t _t = globaltimer(); c.ctl()->subNanos[k] += _t - tRw; tRw = _t; } } while (0)
#else
#define RW_DONE(k) do { } while (0)
#endif
            // room in the block's item list for a warp's items; without it they are counted globally (final slots at once)
            auto reserve = [&](bool valid, bool& forceGlobal) {
                const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
                uint32_t k0 = 0;
                if (laneId() == 0) k0 = atomicAdd(&sh_listCount, (uint32_t)__popc(vmask));
                k0 = __shfl_sync(0xffffffffu, k0, 0);
                forceGlobal = k0 + __popc(vmask) > LIST_CAP;
                if (forceGlobal && laneId() == 0) atomicAdd(&c.ctl()->events[1], 1u);
                return k0 + __popc(vmask & lanemaskLt());
            };
            auto remember = [&](uint32_t i, uint32_t lp, uint32_t slot, uint32_t myk, bool forceGlobal) {
                leafOf[i] = lp;
                if (!forceGlobal) { listItem()[myk] = i; listSlot()[myk] = slot; }       // the final slot is written by passFlush
                else {
                    slotOf[i] = slot;
                    if (myk < LIST_CAP) { listItem()[myk] = 0xffffffffu; listSlot()[myk] = 0; }   // reserved but unused: the warp's items straddled the end of the list
                }
            };
            RW_DONE(12);
            // ---- (1) the items the split phase named (buildWorklist): batch points, and points spilled in earlier rounds. Each sits
            // in a leaf that was split in THIS round (that is how it got on the list), so the step down is the same as in (2):
            // the leaf's record gives the children and the only grid to sample
            // Both loops are software-pipelined: a granule's work is a chain of dependent loads (list entry -> leaf word and
            // point -> grid word -> atomic), and a warp has only a handful of granules, so the list entry two granules ahead and
            // the leaf word + point one granule ahead are in flight while a granule is processed. The grid of the split leaf comes
            // from its record (no side-table load).
            constexpr uint32_t NO_ITEM = 0xffffffffu;
            auto sampleSplitLeaf = [&](uint64_t grid, const Coords& q, uint32_t color, uint32_t node, uint32_t level) {
                if (!nested(q)) atomicOr(&c.ctl()->errorFlags, ERR_FAR_POINT);         // (as sampleUp flags it)
                const uint32_t cell = cellAt(q, level);
                uint32_t* word = reinterpret_cast<uint32_t*>(grid) + (cell >> 5);
                const uint32_t bit = 1u << (cell & 31u);
                const uint32_t seen = (UNCACHED_GRID || SIMLOD_REWALK_L2TEST) ? ldcg(word) : *word;
                if ((seen & bit) == 0 && (atomicOr(word, bit) & bit) == 0) recordVoxel(c, b, node, cell, color);
            };
            {
                const uint32_t stride = rewalkGranuleStride();
                auto loadIndex = [&](uint32_t bs) { const uint32_t u = bs + laneId(); return (bs < numListed && u < numListed) ? wl[u] : NO_ITEM; };
                auto loadItem = [&](uint32_t i, uint32_t& lp, uint4& pt) {
                    lp = 0; pt = make_uint4(0, 0, 0, 0);
                    if (i != NO_ITEM) {
                        pt = i >= scratch::MAX_BATCH ? *reinterpret_cast<const uint4*>(c.spilled() + (i - scratch::MAX_BATCH)) : ldPoint(b.points + i);
                        lp = leafOf[i];
                    }
                };
                uint32_t base = rewalkFirstGranule();
                uint32_t iCur = loadIndex(base), iNext = loadIndex(base + stride);
                uint32_t lpCur; uint4 ptCur;
                loadItem(iCur, lpCur, ptCur);
                for (; base < numListed; base += stride) {
                    uint32_t lpNext; uint4 ptNext;
                    loadItem(iNext, lpNext, ptNext);                                   // granule base + stride
                    const uint32_t iNext2 = loadIndex(base + 2u * stride);
                    const uint32_t i = iCur;
                    const uint4 pt = ptCur;
                    bool valid = i != NO_ITEM;
                    const bool spilledItem = valid && i >= scratch::MAX_BATCH;
                    uint32_t node = 0, level = 0, childBase = 0;
                    uint64_t grid = 0;
                    if (valid) {
                        node = lpCur & 0xffffffu; level = lpCur >> 24;
                        uint32_t k = 0;
                        while (k < numSplit && sh_splitInfo[k].node != node) k++;
                        if (k < numSplit) { childBase = sh_splitInfo[k].childBase; grid = sh_splitInfo[k].grid; }
                        else { valid = false; atomicOr(&c.ctl()->errorFlags, ERR_INTERNAL); }      // cannot happen: listed items sit in split leaves
                        valid = valid && level < SIMLOD_MAX_DEPTH;               // a level-20 node is the leaf even after it "split" (voxels.cu:169)
                    }
                    if (__any_sync(0xffffffffu, valid)) {
                        bool forceGlobal;
                        const uint32_t myk = reserve(valid, forceGlobal);
                        const Coords q = quantize(c, pt);
                        const uint32_t child = childBase + childIndexAt(q, level);
                        if (SAMPLE && valid) sampleSplitLeaf(grid, q, pt.w, node, level);
                        __syncwarp();
                        uint32_t slot = 0;
                        if (COUNT) slot = countInto<true>(c, b, valid, child, level + 1, valid && !spilledItem ? c.runBloom() + (i / perRun) * BLOOM_WORDS : nullptr, forceGlobal);
                        if (valid && COUNT) remember(i, child | ((level + 1) << 24), slot, myk, forceGlobal);
                    }
                    iCur = iNext; lpCur = lpNext; ptCur = ptNext; iNext = iNext2;
                }
            }
            RW_DONE(13);
            // ---- (2) the points spilled in this round, leaf by leaf: a warp's 32 points come out of ONE split leaf, whose
            // record (children, grid, level) is in shared memory — no leaf look-up, no descent: the child is one step down,
            // the only grid on the way is the leaf's own fresh one
            {
                const uint32_t numGranules = sh_splitGranule[numSplit];
                const uint32_t gStride = rewalkGranuleStride() / 32u;
                struct Granule { uint32_t lo, j; bool valid; };
                auto locate = [&](uint32_t g) {
                    Granule r; r.lo = 0; r.j = 0; r.valid = false;
                    if (g < numGranules) {
                        uint32_t lo = 0, hi = numSplit;                      // last split with first granule <= g
                        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (sh_splitGranule[mid] <= g) lo = mid; else hi = mid; }
                        const uint32_t within = (g - sh_splitGranule[lo]) * 32u + laneId();
                        r.lo = lo; r.j = sh_splitInfo[lo].base + within;
                        r.valid = within < sh_splitInfo[lo].stored && sh_splitInfo[lo].level < SIMLOD_MAX_DEPTH;
                    }
                    return r;
                };
                auto loadSpilled = [&](const Granule& gr) { return gr.valid ? *reinterpret_cast<const uint4*>(c.spilled() + gr.j) : make_uint4(0, 0, 0, 0); };
                uint32_t g = rewalkFirstGranule() / 32u;
                Granule cur = locate(g);
                uint4 ptCur = loadSpilled(cur);
                for (; g < numGranules; g += gStride) {
                    const Granule next = locate(g + gStride);
                    const uint4 ptNext = loadSpilled(next);
                    const bool valid = cur.valid;
                    if (__any_sync(0xffffffffu, valid)) {
                        const uint32_t node = sh_splitInfo[cur.lo].node, level = sh_splitInfo[cur.lo].level, childBase = sh_splitInfo[cur.lo].childBase;
                        const uint32_t i = (uint32_t)scratch::MAX_BATCH + cur.j;
                        const uint4 pt = ptCur;
                        bool forceGlobal;
                        const uint32_t myk = reserve(valid, forceGlobal);
                        const Coords q = quantize(c, pt);
                        const uint32_t child = childBase + childIndexAt(q, level);
                        if (SAMPLE && valid) sampleSplitLeaf(sh_splitInfo[cur.lo].grid, q, pt.w, node, level);
                        __syncwarp();
                        uint32_t slot = 0;
                        if (COUNT) slot = countInto(c, b, valid, child, level + 1, nullptr, forceGlobal);
                        if (valid && COUNT) remember(i, child | ((level + 1) << 24), slot, myk, forceGlobal);
                    }
                    cur = next; ptCur = ptNext;
                }
            }
            RW_DONE(14);
        } else {
            if (threadIdx.x == 0) sh_blockLegacy = 1;
            if (first_in_grid()) atomicAdd(&c.ctl()->events[0], 1u);
            // ---- the runs that can hold an item whose leaf was split in the round that just ended: every block published
            // its own run's verdict before the barrier (markAffectedRun), so all blocks build the same list
            if (gridDim.x <= AFFECTED_CAP) {
                const uint32_t* flags = c.runFlag();
                uint32_t numAffected = 0;
                for (uint32_t g0 = 0; g0 < gridDim.x; g0 += blockDim.x) {          // block-uniform trip count
                    const uint32_t g = g0 + threadIdx.x;
                    const uint32_t flag = g < gridDim.x ? ldcg(&flags[g]) : 0u;
                    uint32_t total = 0;
                    const uint32_t off = blockExclusiveScan(flag, total);
                    if (flag) sh_affected[numAffected + off] = g;
                    numAffected += total;
                }
                if (threadIdx.x == 0) sh_numAffected = numAffected;
                __syncthreads();
            }
            // ---- the affected runs and the spilled points as one item space --------------------------------------------
            const Rewalk rw = rewalkSlice(b.size, numSpilled, spilledBefore);
            for (uint32_t base = rewalkFirstGranule(); base < rw.total; base += rewalkGranuleStride()) {
                const uint32_t u = base + laneId();
                uint32_t run = 0xffffffffu, i = 0xffffffffu, node = 0, level = 0;
                bool valid = u < rw.total;
                const bool spilledItem = valid && u >= rw.runItems;
                if (valid) { i = rewalkItem(rw, u, run); valid = spilledItem || i < b.size; }      // (the last run is padded)
                uint4 pt = make_uint4(0, 0, 0, 0);
                if (spilledItem) pt = *reinterpret_cast<const uint4*>(c.spilled() + (i - scratch::MAX_BATCH));     // independent of the leaf look-up
                if (valid) {
                    uint32_t lp = leafOf[i];
                    node = lp & 0xffffffu; level = lp >> 24;
                    // points spilled in the round that just ended sit in a leaf that was split in it: no need to look
                    if (!(spilledItem && i - scratch::MAX_BATCH >= rw.spilledBefore)) valid = c.firstChild()[node] != 0 && level < SIMLOD_MAX_DEPTH;
                }
                if (!__any_sync(0xffffffffu, valid)) continue;
                if (valid && !spilledItem) pt = ldPoint(b.points + i);
                uint32_t lp = 0, slot = 0;
                walk<SAMPLE, COUNT, UNCACHED_GRID, false>(c, b, cache, valid, pt, node, level, level, run != 0xffffffffu ? c.runBloom() + run * BLOOM_WORDS : nullptr, false, lp, slot);
                if (valid && COUNT) { leafOf[i] = lp; slotOf[i] = slot; }
            }

        }
    }
    if (FRESH) {
        // spilled points of this batch, from the root (sampling-only pass after a root split)
        for (uint32_t base = tid - laneId(); base < numSpilled; base += stride) {
            uint32_t j = base + laneId();
            bool valid = j < numSpilled;
            uint4 pt = make_uint4(0, 0, 0, 0);
            if (valid) pt = *reinterpret_cast<const uint4*>(c.spilled() + j);
            uint32_t lp = 0, slot = 0;
            walk<SAMPLE, COUNT, UNCACHED_GRID, true>(c, b, cache, valid, pt, 0, 0, 0, nullptr, false, lp, slot);
        }
    }
    __syncthreads();
}

// flush the block's tables after passItems: one global add per distinct leaf / voxel node (the two tables side by
// side), then block-local ranks -> slots. Must run after waitAllocBlock() when an allocation is in flight.
template <bool SAMPLE, bool COUNT, bool FRESH>
__device__ __forceinline__ void passFlush(const Ctx& c, const Batch& b, uint32_t numSpilled, uint32_t spilledBefore) {
    // (non-FRESH passes: sh_listMode == 1 and no legacy flag means passItems visited the worklist and kept its items in the list)
    if (COUNT && threadIdx.x < VOXTAB_SIZE) {
        uint32_t leaf = sh_leafKey[threadIdx.x], cnt = sh_leafCount[threadIdx.x];
        if (leaf != VOXTAB_EMPTY && cnt > 0) sh_leafBase[threadIdx.x] = countGlobal(c, b, leaf, sh_leafLevel[threadIdx.x], cnt);
    } else if (SAMPLE && threadIdx.x >= 128 && threadIdx.x < 128 + VOXTAB_SIZE) {
        voxelFlushEntry(c, b, threadIdx.x - 128);
    }
    __syncthreads();
    if (SAMPLE) voxelFlushPatch(c, b, FRESH);
    if (COUNT) {
        uint32_t* slotOf = c.slotOf(b.parity);
        if (FRESH) {
            uint32_t blockFirst, blockEnd;
            blockRun(b.size, blockFirst, blockEnd);
            if (blockEnd - blockFirst <= RUNSLOT_CAP) {
                for (uint32_t i = blockFirst + threadIdx.x; i < blockEnd; i += blockDim.x) slotOf[i] = finalSlot(sh_runSlot[i - blockFirst]);
            } else {
                for (uint32_t i = blockFirst + threadIdx.x; i < blockEnd; i += blockDim.x) { uint32_t sl = slotOf[i]; if (sl & PROVISIONAL) slotOf[i] = finalSlot(sl); }
            }
        } else if (sh_roundLegacy == 0) {                                 // the items this block visited in passItems: its list
            const uint32_t n = min(sh_listCount, LIST_CAP);
            const uint32_t* li = listItem();
            const uint32_t* ls = listSlot();
            for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) if (li[k] != 0xffffffffu) slotOf[li[k]] = finalSlot(ls[k]);
        } else {                                                          // ... in the affected runs (legacy rounds)
            const Rewalk rw = rewalkSlice(b.size, numSpilled, spilledBefore);
            for (uint32_t base = rewalkFirstGranule(); base < rw.total; base += rewalkGranuleStride()) {
                const uint32_t u = base + laneId();
                if (u >= rw.total) continue;
                uint32_t run;
                const uint32_t i = rewalkItem(rw, u, run);
                if (u < rw.runItems && i >= b.size) continue;               // padding of the last run
                uint32_t sl = slotOf[i];
                if (sl & PROVISIONAL) slotOf[i] = finalSlot(sl);
            }
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------
// split round, ONE phase (voxels.cu:245-289 spill copy, :308-383 doSplitting). Everything a split
// needs was reserved by the lane that detected it, so for every spilling leaf the jobs are
// independent and spread over the whole grid, one warp per part:
//   parts 0..255    copy a quarter of chunk k of the leaf's stored points into the spill buffer (4 KB, 128-bit, 8 loads in flight per lane)
//   parts 256..287  clear 1/32 of the new inner node's occupancy grid (sic: the root's populated grid too)
//   part  288       create the 8 children, return the chunks to the free stack, publish the node as inner
// ------------------------------------------------------------------------------------------
constexpr uint32_t SPLIT_COPY_PARTS = 256, SPLIT_CLEAR_PARTS = 32, SPLIT_PARTS = SPLIT_COPY_PARTS + SPLIT_CLEAR_PARTS + 1;

__device__ __noinline__ void splitRound(const Ctx c, const Batch b, uint32_t begin, uint32_t end) {
    const uint32_t numWarps = (gridDim.x * blockDim.x) >> 5;
    // the warps of a block take parts that are far apart, so that the copy parts of one leaf spread over all SMs
    const uint32_t warp = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;
    const uint32_t lane = laneId();
    const uint32_t numItems = (end - begin) * SPLIT_PARTS;
    uint32_t* leafOf = c.leafOf(b.parity);
    for (uint32_t item = warp; item < numItems; item += numWarps) {
        const SpillInfo info = c.spill()[begin + item / SPLIT_PARTS];
        const uint32_t part = item % SPLIT_PARTS;
        const uint32_t numChunks = (info.stored + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
        if (part < SPLIT_COPY_PARTS) {
            const uint32_t k = part >> 2, quarter = part & 3u;
            if (k >= numChunks || info.row == 0) continue;
            const Chunk* chunk = reinterpret_cast<const Chunk*>(c.rows()[(uint64_t)(info.row - 1) * scratch::ROW_SLOTS + k]);
            const uint32_t inChunk = min((uint32_t)SIMLOD_POINTS_PER_CHUNK, info.stored - k * SIMLOD_POINTS_PER_CHUNK);
            const uint32_t first = quarter * 256u;                       // points [first, first + 256) of the chunk (the last quarter holds 232)
            const uint32_t n = inChunk > first ? min(256u, inChunk - first) : 0u;
            const uint32_t tag = info.node | (info.level << 24);
            const uint4* src = reinterpret_cast<const uint4*>(&chunk->points[first]);
            const uint32_t dst = info.base + k * SIMLOD_POINTS_PER_CHUNK + first;
#pragma unroll 1
            for (uint32_t h = 0; h < 256u; h += 128u) {                // 4 loads in flight per lane
                uint4 v[4];
#pragma unroll
                for (int u = 0; u < 4; u++) if (h + lane + 32u * u < n) v[u] = src[h + lane + 32u * u];
#pragma unroll
                for (int u = 0; u < 4; u++) if (h + lane + 32u * u < n) {
                    *reinterpret_cast<uint4*>(c.spilled() + dst + h + lane + 32u * u) = v[u];
                    leafOf[scratch::MAX_BATCH + dst + h + lane + 32u * u] = tag;
                }
            }
        } else if (part < SPLIT_COPY_PARTS + SPLIT_CLEAR_PARTS) {
            constexpr uint32_t PER = SIMLOD_GRID_WORDS / 4 / SPLIT_CLEAR_PARTS;       // uint4 per part
            uint4* g = reinterpret_cast<uint4*>(info.grid) + (uint64_t)(part - SPLIT_COPY_PARTS) * PER;
#pragma unroll 4
            for (uint32_t i = lane; i < PER; i += 32) g[i] = make_uint4(0, 0, 0, 0);
        } else {
            Node* parent = &c.nodes[info.node];
            const uint32_t pX = parent->X, pY = parent->Y, pZ = parent->Z;
            if (lane < 8) {
                // default-constructed Node + the fields doSplitting sets (voxels.cu:324-342)
                Node* child = &c.nodes[info.childBase + lane];
                uint64_t* raw = reinterpret_cast<uint64_t*>(child);
#pragma unroll
                for (int w = 0; w < 19; w++) raw[w] = 0;
                child->level = info.level + 1;
                child->X = 2 * pX + ((lane >> 2) & 1);
                child->Y = 2 * pY + ((lane >> 1) & 1);
                child->Z = 2 * pZ + (lane & 1);
                for (int k = 0; k < 20; k++) child->name[k] = parent->name[k];
                reinterpret_cast<uint8_t*>(child)[offsetof(Node, name) + info.level + 1] = (uint8_t)('0' + lane);   // name[level] (sic: level 20 lands on `visible`)
                child->isLeaf = 1;
                parent->children[lane] = child;
                c.firstChild()[info.childBase + lane] = 0;
                c.parentOf()[info.childBase + lane] = info.node;
                c.gridPtr()[info.childBase + lane] = 0;
                c.leafRow()[info.childBase + lane] = 0;
                c.splitState()[info.childBase + lane] = 0;
            }
            // return the leaf's chunks to the free stack (voxels.cu:345-357)
            if (numChunks > 0 && info.row != 0) {
                uint64_t a0 = 0;
                if (lane == 0) a0 = atomicAdd(reinterpret_cast<unsigned long long*>(&c.stats->numAllocatedChunks), (unsigned long long)(0ull - numChunks));
                a0 = __shfl_sync(0xffffffffu, a0, 0);
                for (uint32_t k = lane; k < numChunks && k < scratch::ROW_SLOTS; k += 32) {
                    Chunk* chunk = reinterpret_cast<Chunk*>(c.rows()[(uint64_t)(info.row - 1) * scratch::ROW_SLOTS + k]);
                    chunk->next = nullptr;
                    uint64_t qi = a0 - 1 - k;
                    if (qi < scratch::QUEUE_CAP) c.chunkQueue()[qi] = (uint64_t)chunk;
                    else atomicOr(&c.ctl()->errorFlags, ERR_QUEUE_OVERFLOW);
                }
            }
            __syncwarp();
            if (lane == 0) {
                if (info.row != 0) {                    // the row goes back to the row pool; its contents stay readable for this phase
                    uint32_t f = atomicAdd(&c.ctl()->rowFreeCount, 1u);
                    c.rowFree()[f] = info.row;
                    c.leafRow()[info.node] = 0;
                }
                parent->numPoints = 0;
                parent->points = nullptr;
                parent->grid = reinterpret_cast<SimlodOccupancyGrid*>(info.grid);
                c.gridPtr()[info.node] = info.grid;
                c.firstChild()[info.node] = info.childBase;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// chunk allocation for the nodes touched by a batch (voxels.cu:485-538, 641-672)
// ------------------------------------------------------------------------------------------
// One WARP per touched node, the nodes spread over all warps of the grid (a batch touches a few hundred): the lanes
// fetch / link the node's new chunks side by side, so a node costs a handful of dependent memory round trips
// whatever the number of chunks — the reference walks every node's list with one thread and bumps
// numAllocatedChunks / the heap offset once per chunk (voxels.cu:505-511). The totals, and the pooled-vs-fresh
// split (stack indices >= chunkPoolSize are fresh heap chunks), are the same.
__device__ __noinline__ void allocateChunks(const Ctx c, const Batch b) {
    const uint32_t FULL = 0xffffffffu;
    const uint32_t lane = laneId();
    const uint32_t numWarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t warp = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;        // consecutive nodes go to different SMs
    const uint32_t numDirtyLeaves = ldv(&b.bc->numDirtyLeaves);
    const uint32_t numDirtyVox = ldv(&b.bc->numDirtyVox);
    const uint64_t poolSize = ldv(&c.stats->chunkPoolSize);
    const uint32_t* dirtyLeaves = c.dirtyLeaves(b.parity);
    const uint32_t* dirtyVox = c.dirtyVox(b.parity);

    for (uint32_t d = warp; d < numDirtyLeaves; d += numWarps) {
        const uint32_t n = dirtyLeaves[d];
        if (c.firstChild()[n] != 0) continue;                       // became an inner node in this batch
        Node* node = &c.nodes[n];
        const uint32_t cnt = node->counter, have = node->numPoints;
        if (cnt <= have) continue;
        const uint32_t existing = (have + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
        uint32_t required = (cnt + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
        if (required > scratch::ROW_SLOTS) { if (lane == 0) atomicOr(&c.ctl()->errorFlags, ERR_ROW_OVERFLOW); required = scratch::ROW_SLOTS; }   // insertion drops the excess
        const uint32_t needed = required > existing ? required - existing : 0;       // <= 64
        if (needed > 0) {
            uint64_t a0 = 0, freshOff = 0;
            uint32_t row = 0;
            if (lane == 0) {
                a0 = atomicAdd(reinterpret_cast<unsigned long long*>(&c.stats->numAllocatedChunks), (unsigned long long)needed);
                const uint64_t firstFresh = a0 > poolSize ? a0 : poolSize;          // indices >= poolSize are new heap chunks (voxels.cu:509-515)
                const uint64_t numFresh = a0 + needed > firstFresh ? a0 + needed - firstFresh : 0;
                if (numFresh) freshOff = atomicAdd(reinterpret_cast<unsigned long long*>(&c.heap()->offset), (unsigned long long)(numFresh * SIMLOD_CHUNK_STRIDE));
                row = c.leafRow()[n];
                if (row == 0) {                                 // first chunk of this leaf: take a row (recycled first)
                    uint32_t f = atomicSub(&c.ctl()->rowFreeCount, 1u);
                    if (f >= 1 && f <= scratch::ROW_CAP) {
                        row = c.rowFree()[f - 1];
                    } else {
                        atomicAdd(&c.ctl()->rowFreeCount, 1u);
                        uint32_t r = atomicAdd(&c.ctl()->rowBump, 1u);
                        if (r >= scratch::ROW_CAP) { atomicOr(&c.ctl()->errorFlags, ERR_ROW_OVERFLOW); row = 0; }
                        else row = r + 1;
                    }
                    c.leafRow()[n] = row;
                }
            }
            a0 = __shfl_sync(FULL, a0, 0); freshOff = __shfl_sync(FULL, freshOff, 0); row = __shfl_sync(FULL, row, 0);
            if (row != 0) {
                const uint64_t firstFresh = a0 > poolSize ? a0 : poolSize;
                uint64_t* slots = c.rows() + (uint64_t)(row - 1) * scratch::ROW_SLOTS;
                // lane l owns new chunks l and l + 32; every chunk's `next` is written by its owner only
                uint64_t ch[2] = {0, 0};
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint32_t t = lane + 32u * h;
                    if (t < needed) {
                        const uint64_t idx = a0 + t;
                        ch[h] = idx < poolSize ? c.chunkQueue()[idx] : (uint64_t)(c.heapBytes + freshOff + (idx - firstFresh) * SIMLOD_CHUNK_STRIDE);
                        slots[existing + t] = ch[h];
                    }
                }
                const uint64_t nextA = __shfl_down_sync(FULL, ch[0], 1), firstB = __shfl_sync(FULL, ch[1], 0), nextB = __shfl_down_sync(FULL, ch[1], 1);
                if (lane < needed) reinterpret_cast<Chunk*>(ch[0])->next = reinterpret_cast<Chunk*>(lane + 1 < needed ? (lane == 31 ? firstB : nextA) : 0ull);
                if (lane + 32u < needed) reinterpret_cast<Chunk*>(ch[1])->next = reinterpret_cast<Chunk*>(lane + 33u < needed ? nextB : 0ull);
                if (lane == 0) {
                    if (existing) reinterpret_cast<Chunk*>(slots[existing - 1])->next = reinterpret_cast<Chunk*>(ch[0]);
                    else node->points = reinterpret_cast<Chunk*>(ch[0]);
                }
            }
        }
        if (lane == 0) node->numPoints = cnt;      // slots [have, cnt) were handed out by the counting pass; filled by insertAll
    }

    // voxel lists: always fresh heap memory, never recycled (voxels.cu:652-666), so a node's new chunks are contiguous.
    // (served from the other end of the warp order, so that leaf and voxel-node allocation land on different warps)
    for (uint32_t d = numWarps - 1 - warp; d < numDirtyVox; d += numWarps) {
        const uint32_t n = dirtyVox[d];
        Node* node = &c.nodes[n];
        const uint32_t cnt = node->numVoxels, have = node->numVoxelsStored;
        if (cnt <= have) continue;
        const uint32_t k0 = have / SIMLOD_POINTS_PER_CHUNK;
        const uint32_t nseg = (cnt - 1) / SIMLOD_POINTS_PER_CHUNK - k0 + 1;
        const uint32_t existing = (have + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
        const uint32_t needed = (cnt + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK - existing;
        uint64_t freshOff = 0, tailPtr = 0;
        uint32_t base = 0;
        if (lane == 0) {
            if (needed) freshOff = atomicAdd(reinterpret_cast<unsigned long long*>(&c.heap()->offset), (unsigned long long)((uint64_t)needed * SIMLOD_CHUNK_STRIDE));
            base = atomicAdd(&b.bc->dirCursor, nseg);
            tailPtr = node->voxelChunks ? c.voxelTail()[n] : 0ull;
        }
        freshOff = __shfl_sync(FULL, freshOff, 0); base = __shfl_sync(FULL, base, 0); tailPtr = __shfl_sync(FULL, tailPtr, 0);
        if ((uint64_t)base + nseg > scratch::DIR_CAP) {
            if (lane == 0) { atomicOr(&c.ctl()->errorFlags, ERR_DIR_OVERFLOW); c.voxelDir()[n] = DirEntry{0xffffffffu, 0}; }
            continue;
        }
        uint64_t* chunkDir = c.chunkDir(b.parity);
        const uint32_t j0 = (have % SIMLOD_POINTS_PER_CHUNK != 0) ? 1u : 0u;         // the partly filled tail chunk takes this batch's first voxels
        uint8_t* first = c.heapBytes + freshOff;
        for (uint32_t t = lane; t < needed; t += 32) {
            Chunk* chunk = reinterpret_cast<Chunk*>(first + (uint64_t)t * SIMLOD_CHUNK_STRIDE);
            chunk->next = t + 1 < needed ? reinterpret_cast<Chunk*>(first + (uint64_t)(t + 1) * SIMLOD_CHUNK_STRIDE) : nullptr;
            chunkDir[base + j0 + t] = (uint64_t)chunk;
        }
        if (lane == 0) {
            c.voxelDir()[n] = DirEntry{base, k0};
            if (j0) chunkDir[base] = tailPtr;
            if (needed > 0) {
                if (tailPtr) reinterpret_cast<Chunk*>(tailPtr)->next = reinterpret_cast<Chunk*>(first); else node->voxelChunks = reinterpret_cast<Chunk*>(first);
                c.voxelTail()[n] = (uint64_t)(first + (uint64_t)(needed - 1) * SIMLOD_CHUNK_STRIDE);
            }
            node->numVoxelsStored = cnt;
        }
    }
}

// ------------------------------------------------------------------------------------------
// insertion: every point/voxel already owns (leaf, slot); the leaf's chunk row (points) or the
// per-batch chunk directory (voxels) turns that into an address with two cached lookups
// (voxels.cu:540-639 insertPoints, 674-698 insertVoxels walk slot/1000 list links instead)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ Point* pointSlotAddress(const Ctx& c, uint32_t row, uint32_t slot) {
    const uint32_t k = slot / SIMLOD_POINTS_PER_CHUNK;
    if (row == 0 || k >= scratch::ROW_SLOTS) return nullptr;       // row / node capacity exceeded (flagged): the point is dropped, never misplaced
    Chunk* chunk = reinterpret_cast<Chunk*>(c.rows()[(uint64_t)(row - 1) * scratch::ROW_SLOTS + k]);
    return &chunk->points[slot % SIMLOD_POINTS_PER_CHUNK];
}

__device__ __forceinline__ void insertVoxel(const Ctx& c, uint32_t parity, uint64_t at) {
    uint64_t key = c.vkey(parity)[at];
    uint32_t cell = (uint32_t)(key & 0x1fffffu);
    uint32_t node = (uint32_t)((key >> 21) & 0xfffffu);
    uint32_t vslot = (uint32_t)(key >> 41);
    const Node* nd = &c.nodes[node];
    uint32_t level = nd->level, X = nd->X, Y = nd->Y, Z = nd->Z;
    // cell centre in world space (voxels.cu:103-114; instruction sequence: see fpmath.cuh)
    float nodeSize = fpx::mul_ftz(fpx::ex2(-fpx::u2f(level)), c.size);
    float vx = fpx::add(fpx::fma(nodeSize, fpx::u2f(X), c.minx),
                        fpx::mul_ftz(fpx::mul(nodeSize, fpx::add(fpx::u2f(cell & 127u), 0.5f)), 0.0078125f));
    float vy = fpx::add(fpx::fma(nodeSize, fpx::u2f(Y), c.miny),
                        fpx::mul_ftz(fpx::mul(nodeSize, fpx::add(fpx::u2f((cell >> 7) & 127u), 0.5f)), 0.0078125f));
    float vz = fpx::add(fpx::fma(nodeSize, fpx::u2f(Z), c.minz),
                        fpx::mul_ftz(fpx::mul(nodeSize, fpx::add(fpx::u2f((cell >> 14) & 127u), 0.5f)), 0.0078125f));
    uint4 v = make_uint4(__float_as_uint(vx), __float_as_uint(vy), __float_as_uint(vz), c.vcolor(parity)[at]);
    DirEntry d = c.voxelDir()[node];
    if (d.base == 0xffffffffu) return;                               // directory overflow (flagged)
    Chunk* chunk = reinterpret_cast<Chunk*>(c.chunkDir(parity)[d.base + (vslot / SIMLOD_POINTS_PER_CHUNK - d.k0)]);
    stPoint(&chunk->points[vslot % SIMLOD_POINTS_PER_CHUNK], v);
}

// The insertion work of a batch — its points, its spilled points, its voxels — is one index space handed out in
// tiles from an atomic cursor: insertion shares a phase with the counting of the next batch, whose cost per block
// depends on the data, so blocks that finish counting early take more tiles and the phase ends together.
constexpr uint32_t INSERT_TILE = 1024;      // 4 items per thread

__device__ __noinline__ void insertAll(const Ctx c, const Batch b, uint32_t numSpilled, uint32_t numSharedVoxels) {
    const uint32_t* leafOf = c.leafOf(b.parity);
    const uint32_t* slotOf = c.slotOf(b.parity);
    const uint32_t* leafRow = c.leafRow();
    // voxels: the per-block backlog segments are uneven; prefix sums of the segment fills (in shared memory, every
    // block the same) turn a position in their concatenation into (segment, entry) by binary search
    __shared__ uint32_t sh_segStart[1025];
    __shared__ uint32_t sh_insTile;
    const uint32_t* blockCursor = c.blockCursor(b.parity);
    const bool listed = gridDim.x <= 1024;
    uint32_t segTotal = 0;
    if (listed) {
        for (uint32_t b0 = 0; b0 < gridDim.x; b0 += blockDim.x) {
            uint32_t blk = b0 + threadIdx.x;
            uint32_t v = blk < gridDim.x ? blockCursor[blk] : 0u;
            uint32_t chunkTotal = 0;
            uint32_t off = blockExclusiveScan(v, chunkTotal);
            if (blk < gridDim.x) sh_segStart[blk] = segTotal + off;
            segTotal += chunkTotal;
        }
        if (threadIdx.x == 0) sh_segStart[gridDim.x] = segTotal;
    }
    const uint32_t endPoints = b.size, endSpilled = endPoints + numSpilled, endSeg = endSpilled + segTotal, total = endSeg + numSharedVoxels;

    auto insertOne = [&](uint32_t i) {
        if (i < endSpilled) {
            const bool sp = i >= endPoints;
            const uint32_t item = sp ? (uint32_t)scratch::MAX_BATCH + (i - endPoints) : i;
            uint4 pt = sp ? *reinterpret_cast<const uint4*>(c.spilled() + (i - endPoints)) : ldPoint(b.points + i);
            Point* d = pointSlotAddress(c, leafRow[leafOf[item] & 0xffffffu], slotOf[item]);
            if (d) stPoint(d, pt);
        } else if (i < endSeg) {
            const uint32_t v = i - endSpilled;
            uint32_t lo = 0, hi = gridDim.x;                     // last segment with start <= v
            while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (sh_segStart[mid] <= v) lo = mid; else hi = mid; }
            insertVoxel(c, b.parity, (uint64_t)lo * c.segCap + (v - sh_segStart[lo]));
        } else {
            insertVoxel(c, b.parity, scratch::VOXEL_CAP - scratch::VOXEL_SHARED + (i - endSeg));
        }
    };

    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) sh_insTile = atomicAdd(&b.bc->insertCursor, 1u);
        __syncthreads();
        const uint64_t base64 = (uint64_t)sh_insTile * INSERT_TILE;
        if (base64 >= total) break;
        const uint32_t base = (uint32_t)base64;
        if (base + INSERT_TILE <= endPoints) {
            // a tile of batch points: four independent items per thread, so that the three dependent lookups
            // (item -> leaf row -> chunk) of one overlap with those of the others
            constexpr int U = INSERT_TILE / 256;
            uint4 p[U]; uint32_t n[U], sl[U], r[U]; Point* dst[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const uint32_t i = base + threadIdx.x + 256u * u;
                p[u] = ldPoint(b.points + i);
                n[u] = leafOf[i] & 0xffffffu;
                sl[u] = slotOf[i];
            }
#pragma unroll
            for (int u = 0; u < U; u++) r[u] = leafRow[n[u]];
#pragma unroll
            for (int u = 0; u < U; u++) dst[u] = pointSlotAddress(c, r[u], sl[u]);
#pragma unroll
            for (int u = 0; u < U; u++) if (dst[u]) stPoint(dst[u], p[u]);
        } else {
#pragma unroll 1
            for (uint32_t u = 0; u < INSERT_TILE / 256; u++) {
                const uint32_t i = base + threadIdx.x + 256u * u;
                if (i < total) insertOne(i);
            }
        }
    }
    if (!listed) {       // grids beyond 1024 blocks: every block inserts the voxels of its own segment
        const uint32_t own = blockCursor[blockIdx.x];
        for (uint32_t e = threadIdx.x; e < own; e += blockDim.x) insertVoxel(c, b.parity, (uint64_t)blockIdx.x * c.segCap + e);
    }
    __syncthreads();
}

// The control words every thread needs right after a grid barrier (this batch's counters, the clock, the heap mark, the
// next batch's size). 4 224 warps (H100) loading the same few L2 lines one dependent load after the other serialise on every
// batch; instead one thread per block loads all of them at once (independent loads, two of them 16 bytes wide) and the
// block reads them from shared memory.
struct Snapshot {
    uint32_t numSpillTotal, numSpilled, numBacklog, numDirtyLeaves, numDirtyVox, dirCursor, voxelsCreated, insertCursor;
    uint32_t rootFirstChild, nextBatchSize;
    uint64_t elapsedNanos, memUsed;
};
__shared__ Snapshot sh_snap;
__device__ __forceinline__ void takeSnapshot(const Ctx& c, const BatchCounters* bc, uint32_t parity, const uint32_t* nextBatchSize) {
    if (threadIdx.x == 0) {
        uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
        asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a0), "=r"(a1), "=r"(a2), "=r"(a3) : "l"(bc) : "memory");
        asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3) : "l"(reinterpret_cast<const uint8_t*>(bc) + 16) : "memory");
        const uint64_t el = ldv(&c.ctl()->elapsedByParity[parity]), mu = ldv(&c.ctl()->memUsed);
        const uint32_t fc = ldv(&c.firstChild()[0]);
        const uint32_t nb = nextBatchSize ? ldv(nextBatchSize) : 0u;
        Snapshot sn;
        sn.numSpillTotal = a0; sn.numSpilled = a1; sn.numBacklog = a2; sn.numDirtyLeaves = a3; sn.numDirtyVox = b0; sn.dirCursor = b1; sn.voxelsCreated = b2; sn.insertCursor = b3;
        sn.rootFirstChild = fc; sn.nextBatchSize = nb; sn.elapsedNanos = el; sn.memUsed = mu;
        sh_snap = sn;
    }
    __syncthreads();
}
static_assert(offsetof(BatchCounters, numSpilled) == 4 && offsetof(BatchCounters, numBacklog) == 8 && offsetof(BatchCounters, numDirtyLeaves) == 12 &&
              offsetof(BatchCounters, numDirtyVox) == 16 && offsetof(BatchCounters, voxelsCreated) == 24 && sizeof(BatchCounters) == 32, "takeSnapshot reads BatchCounters as two 16-byte quads");

__device__ __forceinline__ void clearWorklist(Ctl::Worklist* w) { w->cursor[0] = 0; w->cursor[1] = 0; w->legacy = 0; }
__device__ __forceinline__ void clearBatchCounters(BatchCounters* b) {
    b->numSpillTotal = 0; b->numSpilled = 0; b->numBacklog = 0; b->numDirtyLeaves = 0; b->numDirtyVox = 0; b->dirCursor = 0; b->voxelsCreated = 0; b->insertCursor = 0;
}

// Upper bound of what the allocation of a counted batch can still take from the heap (for the capacity guard,
// which the reference evaluates with that batch already allocated, voxels.cu:896-912)
__device__ __forceinline__ uint64_t pendingAllocationBound(const Batch& b) {
    const uint64_t chunks = ((uint64_t)b.size + ldv(&b.bc->numSpilled) + ldv(&b.bc->voxelsCreated)) / SIMLOD_POINTS_PER_CHUNK
                          + ldv(&b.bc->numDirtyLeaves) + ldv(&b.bc->numDirtyVox) + 2;
    return chunks * SIMLOD_CHUNK_STRIDE;
}

// first thread of the grid: what the reference does at the end of a batch (voxels.cu:925-949)
__device__ __forceinline__ void finishBatchBookkeeping(const Ctx& c, const Batch& b, uint64_t tStart) {
    uint64_t allocated = ldv(&c.stats->numAllocatedChunks);
    if (allocated > ldv(&c.stats->chunkPoolSize)) c.stats->chunkPoolSize = allocated;        // voxels.cu:535-537
    c.stats->batchletIndex = b.index + 1;
    c.stats->numPointsProcessed += b.size;
    c.ctl()->spilledTotal += min(ldv(&b.bc->numSpilled), (uint32_t)scratch::SPILL_CAP);
    atomicAdd(reinterpret_cast<unsigned long long*>(&c.ctl()->voxelsTotal), (unsigned long long)min(ldv(&b.bc->numBacklog), (uint32_t)scratch::VOXEL_SHARED));   // other blocks are adding theirs
    c.ctl()->memUsed = ldv(&c.heap()->offset);
}

// ------------------------------------------------------------------------------------------
// kernel_construct — voxels.cu:804-1010
// ------------------------------------------------------------------------------------------
#ifndef SIMLOD_TIMERS
#define SIMLOD_TIMERS 0
#endif
#ifndef SIMLOD_BLOCKS_PER_SM
#define SIMLOD_BLOCKS_PER_SM 4         // tuning knob (tools/exp_variants.py)
#endif
extern "C" __global__ void __launch_bounds__(256, SIMLOD_BLOCKS_PER_SM)
kernel_construct(const Uniforms uniforms, Point* points, uint32_t* buffer, uint8_t* buffer_persistent, Node* nodes,
                 Stats* stats, uint64_t* frameStartTimestamp, CudaPrint* cudaprint,
                 uint32_t* numBatchesUploaded_volatile, uint32_t* batchSizes) {
    cg::grid_group grid = cg::this_grid();
    const bool first = grid.thread_rank() == 0;
    const uint64_t tStart = globaltimer();

    Ctx c;
    c.buf = reinterpret_cast<uint8_t*>(buffer);
    c.nodes = nodes;
    c.stats = stats;
    c.heapBytes = buffer_persistent;
    c.segCap = gridDim.x <= scratch::BLOCK_CAP ? (uint32_t)((scratch::VOXEL_CAP - scratch::VOXEL_SHARED) / gridDim.x) : 0u;
    // octree cube = boxMin + max extent on every axis (voxels.cu:860-863)
    float sx = fpx::sub(uniforms.boxMax[0], uniforms.boxMin[0]);
    float sy = fpx::sub(uniforms.boxMax[1], uniforms.boxMin[1]);
    float sz = fpx::sub(uniforms.boxMax[2], uniforms.boxMin[2]);
    c.size = fmaxf(fmaxf(sx, sy), sz);
    c.rcpSize = fpx::rcp(c.size);
    c.minx = uniforms.boxMin[0]; c.miny = uniforms.boxMin[1]; c.minz = uniforms.boxMin[2];
    Ctl* ctl = c.ctl();

    if (first) {
        *frameStartTimestamp = tStart;
        ctl->numBatchesUploaded = *(volatile uint32_t*)numBatchesUploaded_volatile;   // one snapshot for all threads
        ctl->elapsedNanos = 0; ctl->elapsedByParity[0] = 0; ctl->elapsedByParity[1] = 0;
        ctl->memUsed = c.heap()->offset;
        ctl->allocDone = 0;
        for (int i = 0; i < 3; i++) { clearBatchCounters(&ctl->batch[i]); clearWorklist(&ctl->wl[i]); }
        for (int i = 0; i < 8; i++) ctl->statCounters[i] = 0;
        if (stats->batchletIndex == 0) {       // fresh after the reset kernel: the tree is the root alone
            ctl->errorFlags = 0;
            ctl->spilledTotal = 0; ctl->voxelsTotal = 0; ctl->voxelsByPass[0] = 0; ctl->voxelsByPass[1] = 0;
            for (int i = 0; i < 8; i++) ctl->phaseNanos[i] = 0;
            for (int i = 0; i < 16; i++) ctl->subNanos[i] = 0;
            ctl->launchCount = 0;
            for (int i = 0; i < 4; i++) ctl->events[i] = 0;
            for (int i = 0; i < 12; i++) for (int j = 0; j < 4; j++) ctl->roundHist[i][j] = 0;
            ctl->rowBump = 0; ctl->rowFreeCount = 0;
            c.firstChild()[0] = 0;
            c.parentOf()[0] = 0;
            c.leafRow()[0] = 0;
            c.splitState()[0] = 0;
            c.gridPtr()[0] = (uint64_t)nodes[0].grid;
        }
    }
    if (threadIdx.x == 0) { sh_allocTarget = 0; sh_allocSeen = 0; sh_numAffected = 0; }
    tileBarInit();
    grid.sync();
    uint64_t tPhase = tStart;
    // developer timers (tools/dev_check.py): -DSIMLOD_TIMERS=1 per phase, =2 also block 0's timeline inside the phases.
    // Off in the shipped build: every warp pays for the `first` test at each site.
#if SIMLOD_TIMERS >= 1
#define PHASE_DONE(k) do { if (first) { uint64_t _t = globaltimer(); ctl->phaseNanos[k] += _t - tPhase; tPhase = _t; tSub = _t; } } while (0)
    uint64_t tSub = tStart;
#else
#define PHASE_DONE(k) do { } while (0)
#endif
#if SIMLOD_TIMERS >= 2
#define SUB_DONE(k) do { if (first) { uint64_t _t = globaltimer(); ctl->subNanos[k] += _t - tSub; tSub = _t; } } while (0)
#else
#define SUB_DONE(k) do { } while (0)
#endif
    PHASE_DONE(7);

    const uint32_t numBatchesUploaded = ldv(&ctl->numBatchesUploaded);
    const uint32_t firstBatch = ldv(&stats->batchletIndex);
    const uint32_t numBatches = min(numBatchesUploaded - firstBatch, 20u);     // voxels.cu:883
    const uint32_t lastBatch = firstBatch + numBatches;

    bool havePending = false;          // a counted batch whose allocation + insertion has not run yet
    Batch pending{};
    uint32_t pendingSpilled = 0, pendingBacklog = 0;
    uint64_t pendingBound = 0;         // upper bound of what the pending batch's allocation can still take from the heap (voxels.cu:896-912
                                       // evaluates the capacity guard with that batch already allocated)
    uint32_t allocEpochs = 0;          // in-phase allocations of this launch so far
    auto slotSize = [&](uint32_t batchIndex) { return &batchSizes[batchIndex % SIMLOD_BATCH_STREAM_SIZE]; };

    if (numBatches > 0) takeSnapshot(c, &ctl->batch[firstBatch % 3u], firstBatch & 1u, slotSize(firstBatch));
    for (uint32_t batchIndex = firstBatch; batchIndex < lastBatch; batchIndex++) {
        // (sh_snap: taken after the last barrier — heap mark, clock, root state, this batch's size)
        Batch b;
        const uint32_t ringSlot = batchIndex % SIMLOD_BATCH_STREAM_SIZE;
        b.size = min(sh_snap.nextBatchSize, (uint32_t)SIMLOD_MAX_BATCH_SIZE);
        b.points = points + (uint64_t)ringSlot * SIMLOD_MAX_BATCH_SIZE;
        b.index = batchIndex;
        b.parity = batchIndex & 1u;
        b.bc = &ctl->batch[batchIndex % 3u];

        // capacity guard (voxels.cu:896-912): stop consuming batches 200 MB before the heap is full
        const uint64_t memUsed = sh_snap.memUsed + (havePending ? pendingBound : 0ull);
        const bool memCapacityReached = memUsed + 200000000ull >= uniforms.persistentBufferCapacity;
        if (first) stats->memCapacityReached = memCapacityReached ? 1 : 0;
        if (memCapacityReached) break;

        const bool deferSampling = sh_snap.rootFirstChild == 0;    // root still a leaf: see DESIGN.md §4 (root grid is wiped when it splits)
        const float elapsedMs = float(sh_snap.elapsedNanos) / 1000000.0f;
        if (batchIndex > firstBatch && elapsedMs > 10.0f) break;   // MAX_PROCESSING_TIME (voxels.cu:22,940), as of the end of the previous batch's fused phase

        // ---- fused phase: allocate b-1 | count (+ sample) b | insert b-1 ------------------------------
        SUB_DONE(11);
        if (havePending) {
            allocEpochs++;
            if (threadIdx.x == 0) { sh_allocTarget = allocEpochs * gridDim.x; sh_allocSeen = 0; }
            __syncthreads();
            allocateChunks(c, pending);
            __syncthreads();
            if (threadIdx.x == 0) { __threadfence(); atomicAdd(&ctl->allocDone, 1u); }
        }
        SUB_DONE(0);
        if (first) { clearBatchCounters(&ctl->batch[(batchIndex + 1) % 3u]); clearWorklist(&ctl->wl[(batchIndex + 1) % 3u]); }      // idle set: last used by batch b-2, next by b+1
        if (deferSampling) passItems<false, true, true, false>(c, b, 0, 0, 0);
        else               passItems<true, true, true, false>(c, b, 0, 0, 0);
        SUB_DONE(1);
        waitAllocBlock(c);
        SUB_DONE(2);
        if (deferSampling) passFlush<false, true, true>(c, b, 0, 0);
        else               passFlush<true, true, true>(c, b, 0, 0);
        SUB_DONE(3);
        if (havePending) {
            if (first) finishBatchBookkeeping(c, pending, tStart);          // all allocations of b-1 are complete (waitAllocBlock)
            insertAll(c, pending, pendingSpilled, pendingBacklog);
            if (threadIdx.x == 0) sh_allocTarget = 0;
            havePending = false;
        }
        if (first) { const uint64_t el = globaltimer() - tStart; ctl->elapsedNanos = el; ctl->elapsedByParity[b.parity] = el; }
        SUB_DONE(4);
        grid.sync();
        const uint32_t* nextSize = batchIndex + 1 < lastBatch ? slotSize(batchIndex + 1) : nullptr;
        takeSnapshot(c, b.bc, b.parity, nextSize);
        SUB_DONE(5);
        PHASE_DONE(0);

        // ---- split rounds (voxels.cu:385-415 expand): 2 barriers each ------------------------
        uint32_t spillBegin = 0, spilledBefore = 0;
        for (int round = 0; round < 24; round++) {
            const uint32_t spillEnd = min(sh_snap.numSpillTotal, (uint32_t)scratch::SPILLNODE_CAP);
            if (spillEnd == spillBegin) break;
#if SIMLOD_TIMERS >= 2
            const uint64_t tRound = first ? globaltimer() : 0ull;
#endif
            markAffectedRun(c, b, spillBegin, spillEnd);
            buildWorklist(c, b, spillBegin, spillEnd, (uint32_t)round);
            splitRound(c, b, spillBegin, spillEnd);
            SUB_DONE(6);
            grid.sync();
            SUB_DONE(7);
            PHASE_DONE(1);
#if SIMLOD_TIMERS >= 1
            if (first) ctl->phaseNanos[6] += 1;
#endif
            const uint32_t numSpilled = min(sh_snap.numSpilled, (uint32_t)scratch::SPILL_CAP);     // (reserved when the split was requested: final since the snapshot)
            if (threadIdx.x == 0) {
                Ctl::Worklist* w = &ctl->wl[b.index % 3u];
                const uint32_t lg = ldv(&w->legacy), nl = ldv(&w->cursor[round & 1]);
                sh_roundLegacy = lg; sh_roundListed = nl;
            }
            if (first) ctl->wl[b.index % 3u].cursor[(round + 1) & 1] = 0;       // the list of the previous round has been consumed
            __syncthreads();
            if (deferSampling) passItems<false, true, false, false>(c, b, numSpilled, spilledBefore, (uint32_t)round, spillBegin, spillEnd);
            else               passItems<true, true, false, false>(c, b, numSpilled, spilledBefore, (uint32_t)round, spillBegin, spillEnd);
            SUB_DONE(8);
            if (deferSampling) passFlush<false, true, false>(c, b, numSpilled, spilledBefore);
            else               passFlush<true, true, false>(c, b, numSpilled, spilledBefore);
            SUB_DONE(9);
            grid.sync();
#if SIMLOD_TIMERS >= 2
            if (first) {
                const uint32_t listed = sh_roundLegacy ? 0u : min(sh_roundListed, (uint32_t)scratch::WL_CAP), moved = numSpilled - spilledBefore;
                const uint32_t cls = min(11u, (32u - (uint32_t)__clz(listed + moved)) / 2u);
                ctl->roundHist[cls][0] += 1; ctl->roundHist[cls][1] += globaltimer() - tRound; ctl->roundHist[cls][2] += listed; ctl->roundHist[cls][3] += moved;
            }
#endif
            takeSnapshot(c, b.bc, b.parity, nextSize);
            SUB_DONE(10);
            PHASE_DONE(2);
            spillBegin = spillEnd;
            spilledBefore = numSpilled;
        }
        const uint32_t numSpilled = min(sh_snap.numSpilled, (uint32_t)scratch::SPILL_CAP);
        if (deferSampling) {
            // the root was a leaf when the batch started: sample along the final paths, as the reference does after
            // expand() (voxels.cu:738-742). The root's grid may just have been cleared in place: probe it through L2.
            passItems<true, false, true, true>(c, b, numSpilled, 0, 0);
            passFlush<true, false, true>(c, b, numSpilled, 0);
            grid.sync();
            takeSnapshot(c, b.bc, b.parity, nextSize);
            PHASE_DONE(3);
        }
        havePending = true;
        pending = b;
        pendingSpilled = numSpilled;
        pendingBacklog = min(sh_snap.numBacklog, (uint32_t)scratch::VOXEL_SHARED);
        pendingBound = (((uint64_t)b.size + sh_snap.numSpilled + sh_snap.voxelsCreated) / SIMLOD_POINTS_PER_CHUNK + sh_snap.numDirtyLeaves + sh_snap.numDirtyVox + 2) * SIMLOD_CHUNK_STRIDE;
    }

    // ---- the last counted batch: allocate, then insert ------------------------------------------
    if (havePending) {
        allocateChunks(c, pending);
        grid.sync();
        PHASE_DONE(4);
        if (first) finishBatchBookkeeping(c, pending, tStart);
        insertAll(c, pending, pendingSpilled, pendingBacklog);
    }

    // ---- octree statistics (voxels.cu:958-1009), same phase as the last insertion --------------------
    {
        const uint32_t numNodes = min(ldv(&stats->numNodes), (uint32_t)scratch::NODE_CAP);
        const uint32_t stride = gridDim.x * blockDim.x;
        uint32_t inner = 0, leaves = 0, nonempty = 0, pts = 0, vox = 0, chP = 0, chV = 0;
        for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < numNodes; n += stride) {
            const Node* node = &nodes[n];
            if (c.firstChild()[n] == 0) {
                uint32_t np = node->numPoints;
                leaves++; pts += np; chP += (np + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
                if (np > 0) nonempty++;
            } else {
                uint32_t nv = node->numVoxels;
                inner++; vox += nv; chV += (nv + SIMLOD_POINTS_PER_CHUNK - 1) / SIMLOD_POINTS_PER_CHUNK;
            }
        }
        uint32_t vals[7] = {inner, leaves, nonempty, pts, vox, chP, chV};
#pragma unroll
        for (int k = 0; k < 7; k++) {
            uint32_t v = vals[k];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (laneId() == 0 && v) atomicAdd(&ctl->statCounters[k], v);
        }
    }
    grid.sync();
    PHASE_DONE(5);
    if (first) {
        stats->numInner = ldv(&ctl->statCounters[0]);
        stats->numLeaves = ldv(&ctl->statCounters[1]);
        stats->numNonemptyLeaves = ldv(&ctl->statCounters[2]);
        stats->numPoints = ldv(&ctl->statCounters[3]);
        stats->numVoxels = ldv(&ctl->statCounters[4]);
        stats->numChunksPoints = ldv(&ctl->statCounters[5]);
        stats->numChunksVoxels = ldv(&ctl->statCounters[6]);
        stats->allocatedBytes_momentary = scratch::TOTAL;
        stats->allocatedBytes_persistent = ldv(&c.heap()->offset);
        stats->frameID = (uint32_t)uniforms.frameCounter;
        stats->dbg = ldv(&ctl->errorFlags);
        const uint32_t lc = ctl->launchCount++;
        ctl->launchClock[lc & 31u][0] = tStart; ctl->launchClock[lc & 31u][1] = globaltimer();
    }
}
