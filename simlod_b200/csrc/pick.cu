// pick.cu — the sample under each pixel: for every pixel of the frame kernel_render draws, the drawn sample that wins it,
// as an index into the view export's sample array (DESIGN.md §9.9).
//
// The view export's plan (simlod_export_view_flags, simlod_export_plan_view, simlod_export_collect in export.cu) lists
// the drawn nodes' chunks as items whose `dst` is the export index of their first sample. Then:
//
//   simlod_pick_clear   both frames: key = the limit a hit must stay below, index = none; the hit counter = 0
//   simlod_pick_key     a warp per item: every sample is projected and coloured with kernel_render's own sequence
//                       (splat.cuh) and splatted over the pixels the renderer covers, by an early-out compare and a 64-bit
//                       atomicMin of its key depth << 32 | colour
//   simlod_pick_index   the same walk: a sample whose key equals a covered pixel's takes an atomicMin of its export index,
//                       so a tie on the key goes to the lowest index whatever order the atomics land in
//   simlod_pick_write   the whole frame or a list of pixels: the index (-1 for none) and, optionally, the sample itself
//
// Reads the ABI, the export scratch and its own two frames; writes nothing else but the destinations.
#include <stdint.h>
#include "../../include/simlod_abi.h"
#include "splat.cuh"
#include "export_common.cuh"
#include "region.cuh"

constexpr uint64_t NO_INDEX = ~0ull;
constexpr uint32_t PICK_UNROLL = 4;

// A pixel is hit when its winning key is below the value the frame is cleared to (depth +inf, colour 0x00332211); with
// HQS, when the winner's depth is below +inf (the depth target is cleared to +inf, the colour does not compete).
__device__ __forceinline__ uint64_t hitLimit(const SimlodUniforms& u) {
    return u.useHighQualityShading ? 0x7f800000ull << 32 : (0x7f800000ull << 32) | 0x00332211ull;
}

extern "C" __global__ void __launch_bounds__(256)
simlod_pick_clear(const SimlodUniforms u, const PickArgs a) {
    const uint32_t numPixels = (uint32_t)(fpx::f2i(u.width) * fpx::f2i(u.height));
    const uint64_t limit = hitLimit(u);
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < numPixels; p += gridDim.x * blockDim.x) {
        a.key[p] = limit;
        a.index[p] = NO_INDEX;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *a.hits = 0;
}

// The key pass (indexPass false) and the index pass (true). The candidates, their keys and the pixels they cover are
// kernel_render's (render.cu, all four draw paths): project(), inside (and depth > 0 with HQS), sampleColor() with the
// record's level and node colour id, pixels clamp(x + ox, 0, W) + W clamp(y + oy, 0, H) for 0 <= ox, oy < pointSize.
// Ids >= W*H lie outside the frame (the renderer's stores there land behind it) and are dropped. A sample the clip drops
// (region.cuh clipKeeps, as simlod_render_clip tests it) is no candidate.
template <bool indexPass>
__device__ __forceinline__ void pickPass(const SimlodUniforms& u, const PickArgs& a) {
    if (!u.showPoints) return;
    const bool hqs = u.useHighQualityShading != 0;
    const uint64_t limit = hitLimit(u);
    const int width = fpx::f2i(u.width), height = fpx::f2i(u.height);
    const uint32_t numPixels = (uint32_t)(width * height);
    const int pointSize = u.pointSize;
    const SimlodFloat4* T = u.transform.rows;
    const Item* items = reinterpret_cast<const Item*>(a.items);
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t numWarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t k = warp; k < a.numItems; k += numWarps) {
        const Item it = items[k];
        const SimlodExportNode* r = a.rec + itemRecord(k, a.recItem, a.numRecords);
        const uint32_t level = r->level, colorId = nodeColorId(r);
        const uint4* src = reinterpret_cast<const uint4*>(it.src);
        const uint64_t first = it.dst & 0xffffffffffffull;
        const uint32_t count = (uint32_t)(it.dst >> 48);
        for (uint32_t b = 0; b < count; b += 32 * PICK_UNROLL) {
            uint4 v[PICK_UNROLL];
#pragma unroll
            for (uint32_t s = 0; s < PICK_UNROLL; s++) {
                const uint32_t j = b + s * 32 + lane;
                if (j < count) v[s] = src[j];
            }
#pragma unroll
            for (uint32_t s = 0; s < PICK_UNROLL; s++) {
                const uint32_t j = b + s * 32 + lane;
                if (j >= count || !clipKeeps(a.clip, __uint_as_float(v[s].x), __uint_as_float(v[s].y), __uint_as_float(v[s].z))) continue;
                const Projected pr = project(T, u.width, u.height, __uint_as_float(v[s].x), __uint_as_float(v[s].y), __uint_as_float(v[s].z));
                if (!pr.inside || (hqs && !(pr.depth > 0.0f))) continue;
                const uint64_t key = ((uint64_t)__float_as_uint(pr.depth) << 32) | sampleColor(u, v[s].w, level, colorId);
                if (key >= limit) continue;
                const uint64_t index = first + j;
                for (int ox = 0; ox < pointSize; ox++)
                for (int oy = 0; oy < pointSize; oy++) {
                    const uint32_t qx = (uint32_t)max(0, min(pr.x + ox, width));
                    const uint32_t qy = (uint32_t)max(0, min(pr.y + oy, height));
                    const uint32_t p = qx + (uint32_t)width * qy;
                    if (p >= numPixels) continue;
                    if (!indexPass) {
                        if (key < a.key[p]) atomicMin(reinterpret_cast<unsigned long long*>(&a.key[p]), (unsigned long long)key);
                    } else if (key == a.key[p] && index < a.index[p]) {
                        atomicMin(reinterpret_cast<unsigned long long*>(&a.index[p]), (unsigned long long)index);
                    }
                }
            }
        }
    }
}

// Both passes are declared with 2 blocks per SM: with the block size alone ptxas keeps them at 40 registers and spills.
extern "C" __global__ void __launch_bounds__(256, 2)
simlod_pick_key(const SimlodUniforms u, const PickArgs a) {
    pickPass<false>(u, a);
}

extern "C" __global__ void __launch_bounds__(256, 2)
simlod_pick_index(const SimlodUniforms u, const PickArgs a) {
    pickPass<true>(u, a);
}

// n pixels: pixel t is pixels[t], or t when there is no list. dstIndex[t] = its sample index or -1; dstSamples[t] (when
// given) = that sample, found by binary search over the items' first indices (items are in index order), or zeros.
extern "C" __global__ void __launch_bounds__(256)
simlod_pick_write(const PickArgs a, const uint32_t* __restrict__ pixels, uint32_t n, int64_t* __restrict__ dstIndex,
                  uint4* __restrict__ dstSamples) {
    const Item* items = reinterpret_cast<const Item*>(a.items);
    uint32_t hits = 0;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const uint64_t index = a.index[pixels ? pixels[t] : t];
        const bool hit = index != NO_INDEX;
        hits += hit ? 1u : 0u;
        if (dstIndex) dstIndex[t] = hit ? (int64_t)index : -1ll;
        if (dstSamples) {
            uint4 v = make_uint4(0, 0, 0, 0);
            if (hit) {
                uint64_t lo = 0, hi = a.numItems;       // the last item whose first index is <= index
                while (hi - lo > 1) {
                    const uint64_t mid = (lo + hi) >> 1;
                    if ((items[mid].dst & 0xffffffffffffull) <= index) lo = mid; else hi = mid;
                }
                v = reinterpret_cast<const uint4*>(items[lo].src)[index - (items[lo].dst & 0xffffffffffffull)];
            }
            dstSamples[t] = v;
        }
    }
    hits = __reduce_add_sync(0xffffffffu, hits);
    if ((threadIdx.x & 31u) == 0 && hits) atomicAdd(reinterpret_cast<unsigned long long*>(a.hits), (unsigned long long)hits);
}
