// construct_layout.cuh — the layout of kernel_construct's scratch ("momentary") buffer: the offsets of every table, the
// control block and the records the builder keeps there. Shared by construct.cu and by the octree import (import.cu),
// which fills the builder's persistent side tables for a loaded octree (DESIGN.md §2, §9.7).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/simlod_abi.h"

// The capacity guard (voxels.cu:896-912): kernel_construct stops consuming batches once the heap offset plus this many
// bytes reaches the persistent buffer's capacity, and a loaded octree must leave them free as well.
constexpr uint64_t HEAP_GUARD_BYTES = 200000000ull;

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
    uint64_t memUsed;              // heap offset for the capacity guard: >= H_j and <= H_j + the grids of batch j, where H_j is the offset
                                   // after batches [0, j) (written by the grid's first thread where no other block can be reading it)
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
    uint64_t heapExact;            // @1392 the heap offset between the two barriers of the capacity guard's exact path
    uint64_t freshBytes;           // @1400 heap bytes taken by the chunk allocation in progress (checked against its bound)
};
static_assert(offsetof(Ctl, roundHist) == 1008 && offsetof(Ctl, freshBytes) == 1400 && sizeof(Ctl) <= 4096, "tools read Ctl by offset; the control block is 4 KB");
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
