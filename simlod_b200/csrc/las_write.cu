// las_write.cu — LAS point records encoded on the GPU (DESIGN.md §9.13): the writer behind simlod_write_las.
//
// las.cu's TMA decode in reverse. Every block iteration takes a tile of 256 16-byte samples with coalesced loads,
// quantises each coordinate in IEEE double exactly as the file contract states, and builds the 26-byte point-format-2
// records in shared memory. Records are only 2-byte aligned, so every field is written as 16-bit halves. A full tile
// (256 x 26 = 6656 bytes, a multiple of 16) leaves shared memory with ONE cp.async.bulk store; the tile's two stages
// let the store of one tile overlap the encode of the next. The ragged last tile of a window is stored with plain
// 16-bit stores.
//
// Each block reduces the per-axis min / max of q over its valid samples and the first invalid source index, then
// issues one atomic each into LasWriteCtl, which the host resets once per call and reads with every window.
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "kernel_args.h"

constexpr uint32_t TILE_HALVES = LAS_WRITE_TILE * LAS_WRITE_RECORD / 2;
static_assert((LAS_WRITE_TILE * LAS_WRITE_RECORD) % 16 == 0, "a full tile is a whole number of 16-byte units");

// q = rint(((double(p) + t) - o) / s), every operation rounded to nearest, half to even; false when q is not an int32
// (a non-finite p gives a non-finite quotient, which fails the range test, as does a NaN)
__device__ __forceinline__ bool quantise(float p, double s, double o, double t, int32_t& q) {
    const double r = rint(__ddiv_rn(__dsub_rn(__dadd_rn((double)p, t), o), s));
    const bool ok = r >= -2147483648.0 && r <= 2147483647.0;
    q = ok ? (int32_t)r : 0;
    return ok;
}

extern "C" __global__ void __launch_bounds__(LAS_WRITE_TILE)
simlod_las_encode(const LasEncodeArgs a) {
    __shared__ __align__(128) uint16_t sh_rec[2][TILE_HALVES];
    __shared__ uint32_t sh_min[6];
    __shared__ unsigned long long sh_invalid;
    if (threadIdx.x < 6) sh_min[threadIdx.x] = ~0u;
    if (threadIdx.x == 0) sh_invalid = ~0ull;
    uint32_t qmin[3] = {~0u, ~0u, ~0u}, qmaxInv[3] = {~0u, ~0u, ~0u};
    unsigned long long invalid = ~0ull;
    const uint64_t numTiles = (a.count + LAS_WRITE_TILE - 1) / LAS_WRITE_TILE;
    uint32_t stage = 0;
    for (uint64_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x, stage ^= 1) {
        const uint64_t first = tile * LAS_WRITE_TILE;
        const uint32_t n = (uint32_t)min((uint64_t)LAS_WRITE_TILE, a.count - first);
        // the bulk store issued from this stage two tiles ago has finished reading it
        if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        __syncthreads();
        uint16_t* r = sh_rec[stage] + threadIdx.x * (LAS_WRITE_RECORD / 2);
        if (threadIdx.x < n) {
            const uint4 v = __ldcs(reinterpret_cast<const uint4*>(a.samples) + first + threadIdx.x);
            int32_t q[3];
            bool ok = quantise(__uint_as_float(v.x), a.scale[0], a.offset[0], a.translation[0], q[0]);
            ok &= quantise(__uint_as_float(v.y), a.scale[1], a.offset[1], a.translation[1], q[1]);
            ok &= quantise(__uint_as_float(v.z), a.scale[2], a.offset[2], a.translation[2], q[2]);
            if (ok) {
                #pragma unroll
                for (int k = 0; k < 3; k++) {
                    const uint32_t u = (uint32_t)q[k] ^ 0x80000000u;
                    qmin[k] = min(qmin[k], u);
                    qmaxInv[k] = min(qmaxInv[k], ~u);
                }
            } else {
                invalid = min(invalid, (unsigned long long)(a.first + first + threadIdx.x));
            }
            #pragma unroll
            for (int k = 0; k < 3; k++) { r[2 * k] = (uint16_t)((uint32_t)q[k] & 0xffffu); r[2 * k + 1] = (uint16_t)((uint32_t)q[k] >> 16); }
            r[6] = 0;                                   // intensity
            r[7] = 0x0009;                              // return 1 of 1; classification 0
            r[8] = 0;                                   // scan angle, user data
            r[9] = 0;                                   // point source ID
            r[10] = (uint16_t)(257u * (v.w & 0xffu));
            r[11] = (uint16_t)(257u * ((v.w >> 8) & 0xffu));
            r[12] = (uint16_t)(257u * ((v.w >> 16) & 0xffu));
        }
        // the generic-proxy writes above become visible to the bulk copy (async proxy)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        uint8_t* dst = a.records + first * LAS_WRITE_RECORD;
        if (n == LAS_WRITE_TILE) {
            if (threadIdx.x == 0) {
                const uint32_t src = (uint32_t)__cvta_generic_to_shared(sh_rec[stage]);
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                             :: "l"(dst), "r"(src), "r"(LAS_WRITE_TILE * LAS_WRITE_RECORD) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        } else {                                        // the window's ragged last tile
            for (uint32_t h = threadIdx.x; h < n * (LAS_WRITE_RECORD / 2); h += blockDim.x)
                reinterpret_cast<uint16_t*>(dst)[h] = sh_rec[stage][h];
        }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    // the block's bounds and first invalid index, then one atomic each
    #pragma unroll
    for (int k = 0; k < 3; k++) {
        qmin[k] = __reduce_min_sync(0xffffffffu, qmin[k]);
        qmaxInv[k] = __reduce_min_sync(0xffffffffu, qmaxInv[k]);
    }
    __syncthreads();
    if ((threadIdx.x & 31u) == 0) {
        #pragma unroll
        for (int k = 0; k < 3; k++) { atomicMin(&sh_min[k], qmin[k]); atomicMin(&sh_min[3 + k], qmaxInv[k]); }
    }
    if (invalid != ~0ull) atomicMin(&sh_invalid, invalid);
    __syncthreads();
    if (threadIdx.x < 3) { if (sh_min[threadIdx.x] != ~0u) atomicMin(&a.ctl->qmin[threadIdx.x], sh_min[threadIdx.x]); }
    else if (threadIdx.x < 6) { if (sh_min[threadIdx.x] != ~0u) atomicMin(&a.ctl->qmaxInv[threadIdx.x - 3], sh_min[threadIdx.x]); }
    else if (threadIdx.x == 6 && sh_invalid != ~0ull) atomicMin(reinterpret_cast<unsigned long long*>(&a.ctl->firstInvalid), sh_invalid);
}
