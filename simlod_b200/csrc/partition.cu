// partition.cu — spatial exchange for a merged multi-GPU octree (SURVEY.md §8f-3).
//
// The reference builds one octree on one GPU. To build ONE octree over G GPUs every rank owns the
// octree cells of a fixed level L (8^L cells of the global cube) that a plan assigns to it, and every
// point travels to the owner of its cell before it is inserted there. These kernels are the sending
// side: a stable partition of a batch by owner whose scatter pass writes each point straight to its
// destination — the owner's receive buffer mapped over NVLink (peer memory) or a local staging
// buffer — so the exchange is the partition's own store stream and no separate copy follows.
//
// The owner of a point is decided with exactly the arithmetic the builder uses to descend
// (construct.cu quantize / childIndexAt = voxels.cu:148-155,171-179), so a point can never reach a
// rank whose cells do not contain it.
//
//   simlod_partition_count    per-block histogram over destination ranks (+ global per-cell histogram)
//   simlod_partition_scan     exclusive scan of the block histograms per destination, totals
//   simlod_partition_scatter  stable scatter: dst[d][offset[d] + rank of the point among the batch's
//                             points for d] = point      (16-byte stores, local or peer); the last block to
//                             finish then releases a flag in every destination ("my bucket has landed")
//   simlod_partition_wait     acquire side: spins until every sender's flag has reached the step's value
#include <stdint.h>
#include "fpmath.cuh"
#include "kernel_args.h"        // PartitionParams, ScatterTargets, CompositeArgs, SignalArgs

using part::MAX_RANKS;
using part::MAX_CELLS;
using part::BLOCK;
constexpr uint32_t WARPS = BLOCK / 32;

__device__ __forceinline__ uint32_t cellOf(const PartitionParams& p, float rcpSize, uint4 pt) {
    float dx = fpx::add(__uint_as_float(pt.x), -p.minx);
    float dy = fpx::add(__uint_as_float(pt.y), -p.miny);
    float dz = fpx::add(__uint_as_float(pt.z), -p.minz);
    uint32_t X = fpx::f2u(fpx::mul_ftz(fpx::mul(dx, 1048576.0f), rcpSize));
    uint32_t Y = fpx::f2u(fpx::mul_ftz(fpx::mul(dy, 1048576.0f), rcpSize));
    uint32_t Z = fpx::f2u(fpx::mul_ftz(fpx::mul(dz, 1048576.0f), rcpSize));
    uint32_t cell = 0;
    for (uint32_t l = 0; l < p.level; l++) {
        uint32_t sh = 19u - l;              // voxels.cu:171-179: bit (19 - level) of each axis, child = x<<2 | y<<1 | z
        cell = (cell << 3) | (((X >> sh) & 1u) << 2) | (((Y >> sh) & 1u) << 1) | ((Z >> sh) & 1u);
    }
    return cell;
}

__device__ __forceinline__ uint4 ldPoint(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

extern "C" __global__ void __launch_bounds__(BLOCK)
simlod_partition_count(const PartitionParams p, const uint4* __restrict__ points, uint32_t* __restrict__ blockHist /*[gridDim][8]*/,
                       uint32_t* __restrict__ cellCounts /*[512], accumulated*/) {
    __shared__ uint32_t sh_cell[MAX_CELLS];
    const uint32_t numCells = 1u << (3u * p.level);
    for (uint32_t i = threadIdx.x; i < numCells; i += BLOCK) sh_cell[i] = 0;
    __syncthreads();
    const float rcpSize = fpx::rcp(p.size);
    const uint32_t first = blockIdx.x * p.perBlock;
    const uint32_t end = min(first + p.perBlock, p.count);
    for (uint32_t i = first + threadIdx.x; i < end; i += BLOCK) {
        const uint32_t cell = cellOf(p, rcpSize, ldPoint(points + i));
        const uint32_t peers = __match_any_sync(__activemask(), cell);          // coherent scans: few distinct cells per warp
        if ((threadIdx.x & 31u) == (uint32_t)__ffs(peers) - 1u) atomicAdd(&sh_cell[cell], (uint32_t)__popc(peers));
    }
    __syncthreads();
    __shared__ uint32_t sh_rank[MAX_RANKS];
    if (threadIdx.x < MAX_RANKS) sh_rank[threadIdx.x] = 0;
    __syncthreads();
    for (uint32_t c = threadIdx.x; c < numCells; c += BLOCK) {
        const uint32_t n = sh_cell[c];
        if (n) { atomicAdd(&sh_rank[p.owner[c]], n); atomicAdd(&cellCounts[c], n); }
    }
    __syncthreads();
    if (threadIdx.x < MAX_RANKS) blockHist[blockIdx.x * MAX_RANKS + threadIdx.x] = sh_rank[threadIdx.x];
}

// one block, warp d scans destination d over the blocks
extern "C" __global__ void __launch_bounds__(BLOCK)
simlod_partition_scan(const uint32_t* __restrict__ blockHist, uint32_t numBlocks, uint32_t* __restrict__ blockBase /*[numBlocks][8]*/,
                      uint32_t* __restrict__ totals /*[8]*/) {
    const uint32_t d = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    uint32_t running = 0;
    for (uint32_t b0 = 0; b0 < numBlocks; b0 += 32) {
        const uint32_t b = b0 + lane;
        const uint32_t v = b < numBlocks ? blockHist[b * MAX_RANKS + d] : 0u;
        uint32_t incl = v;
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += t; }
        if (b < numBlocks) blockBase[b * MAX_RANKS + d] = running + incl - v;
        running += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) totals[d] = running;
}

extern "C" __global__ void __launch_bounds__(BLOCK)
simlod_partition_scatter(const PartitionParams p, const ScatterTargets t, const uint4* __restrict__ points,
                         const uint32_t* __restrict__ blockBase, uint32_t* __restrict__ blocksDone) {
    __shared__ uint32_t sh_warpBuf[2][WARPS][MAX_RANKS];   // points of warp w for destination d in the current 256-point group
                                                            // (two copies by iteration parity: zeroing never races the previous readers)
    __shared__ uint32_t sh_running[MAX_RANKS];          // points of this block already placed per destination
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    if (threadIdx.x < MAX_RANKS) sh_running[threadIdx.x] = blockBase[blockIdx.x * MAX_RANKS + threadIdx.x];
    const float rcpSize = fpx::rcp(p.size);
    const uint32_t first = blockIdx.x * p.perBlock;
    const uint32_t end = min(first + p.perBlock, p.count);
    uint32_t parity = 0;
    for (uint32_t base = first; base < end; base += BLOCK, parity ^= 1u) {            // block-uniform trip count
        uint32_t (*sh_warp)[MAX_RANKS] = sh_warpBuf[parity];
        const uint32_t i = base + threadIdx.x;
        const bool valid = i < end;
        uint4 pt = make_uint4(0, 0, 0, 0);
        uint32_t dst = 0xffffffffu;
        if (valid) { pt = ldPoint(points + i); dst = p.owner[cellOf(p, rcpSize, pt)]; }
        const uint32_t peers = __match_any_sync(0xffffffffu, dst);
        const uint32_t before = (uint32_t)__popc(peers & ((1u << lane) - 1u));     // stable: lanes are in input order
        if (threadIdx.x < WARPS * MAX_RANKS) (&sh_warp[0][0])[threadIdx.x] = 0;
        __syncthreads();
        if (valid && before == 0) sh_warp[warp][dst] = (uint32_t)__popc(peers);
        __syncthreads();
        if (valid) {
            uint32_t pos = sh_running[dst] + before;
            for (uint32_t w = 0; w < warp; w++) pos += sh_warp[w][dst];
            uint4* out = reinterpret_cast<uint4*>(t.ptr[dst]) + t.offset[dst] + pos;
            asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(out), "r"(pt.x), "r"(pt.y), "r"(pt.z), "r"(pt.w) : "memory");
        }
        __syncthreads();
        if (threadIdx.x < MAX_RANKS) {
            uint32_t add = 0;
            for (uint32_t w = 0; w < WARPS; w++) add += sh_warp[w][threadIdx.x];
            sh_running[threadIdx.x] += add;
        }
        // the next iteration's first __syncthreads orders this update before its readers
    }
    // ---- "my buckets have landed": every thread orders its (possibly remote) stores at system scope, the last block
    // to arrive releases this sender's flag in every destination (the threadfence-reduction pattern, system scope)
    if (t.signal[0] != 0) {
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t arrived = atomicAdd(blocksDone, 1u);
            if (arrived == gridDim.x - 1u) {
                __threadfence_system();
                for (uint32_t d = 0; d < p.numRanks; d++)
                    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(t.signal[d]), "r"(t.signalValue) : "memory");
                *blocksDone = 0;
            }
        }
    }
}

// acquire side, one thread per sender: flags[s] >= value  <=>  sender s's stores of this step are visible here.
// Gives up after `timeoutCycles` SM clocks (a peer died) and reports it instead of hanging the stream.
extern "C" __global__ void simlod_partition_wait(const uint32_t* flags, uint32_t numRanks, uint32_t value, uint64_t timeoutCycles,
                                                 uint32_t* __restrict__ timedOut) {
    if (threadIdx.x >= numRanks) return;
    const long long start = clock64();
    for (;;) {
        uint32_t v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
        if ((int32_t)(v - value) >= 0) return;
        if ((uint64_t)(clock64() - start) > timeoutCycles) { atomicExch(timedOut, 1u + threadIdx.x); return; }
        __nanosleep(200);
    }
}

// ------------------------------------------------------------------------------------------------------
// Depth compositing of the ranks' packed framebuffers (DESIGN.md §8/§9.3): the u64 word is depth<<32 | colour, so an
// element-wise unsigned minimum over the ranks is exactly the depth test one GPU's atomicMin performs on the union
// of the samples (render.cu drawPoint = render.cu:61-104 of the reference). Two-shot all-reduce over peer memory in
// ONE kernel: rank r reduces slice r of every rank's buffer (peer loads) and stores the result into slice r of every
// rank's buffer (peer stores); slices are disjoint, so no rank reads what another writes. Ends like the scatter:
// the last block releases this rank's flag in every peer.

extern "C" __global__ void __launch_bounds__(BLOCK)
simlod_composite_min(const CompositeArgs a, uint32_t* __restrict__ blocksDone) {
    const uint64_t lo = a.numWords * a.rank / a.numRanks, hi = a.numWords * (a.rank + 1) / a.numRanks;
    for (uint64_t i = lo + (uint64_t)blockIdx.x * BLOCK + threadIdx.x; i < hi; i += (uint64_t)gridDim.x * BLOCK) {
        unsigned long long m = 0xffffffffffffffffull;
        for (uint32_t s = 0; s < a.numRanks; s++) {
            unsigned long long v;
            asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(reinterpret_cast<const unsigned long long*>(a.fb[s]) + i) : "memory");
            m = v < m ? v : m;
        }
        for (uint32_t d = 0; d < a.numRanks; d++)
            asm volatile("st.relaxed.sys.global.u64 [%0], %1;" :: "l"(reinterpret_cast<unsigned long long*>(a.fb[d]) + i), "l"(m) : "memory");
    }
    if (a.signal[0] != 0) {
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t arrived = atomicAdd(blocksDone, 1u);
            if (arrived == gridDim.x - 1u) {
                __threadfence_system();
                for (uint32_t d = 0; d < a.numRanks; d++)
                    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(a.signal[d]), "r"(a.signalValue) : "memory");
                *blocksDone = 0;
            }
        }
    }
}

// "what this stream has written so far is ready": releases this rank's flag in every peer (enqueued behind the work
// it announces, e.g. the copy of the framebuffer into the peer-visible buffer)
extern "C" __global__ void simlod_peer_signal(const SignalArgs a) {
    if (threadIdx.x < a.numRanks) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(a.signal[threadIdx.x]), "r"(a.value) : "memory");
    }
}
