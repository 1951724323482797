// render_layout.cuh — the layout of kernel_render's buffer ("renderbuffer"). Shared by render.cu and by the host, which
// sizes the buffer and reads the framebuffer back from it.
#pragma once
#include <stdint.h>

// The framebuffer and the HQS targets sit where the reference's bump allocator puts them (render.cu:1108-1123,172,224-231),
// so both kernels can be read back with the same offsets; the area the reference uses for 100 000 Node copies holds our
// work queue, and the unused tail of the 200 000 000-byte buffer (main.cpp:556) a cache of the nodes' chunk lists.
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

// The end of the targets of a frame of `numPixels` pixels: the u64 framebuffer, then the HQS targets as kernel_render
// places them (render.cu:172,224-231 of the reference: a 4-byte counter rounded to 16, u32 depth, 4 x u32 colour sums).
constexpr uint64_t targetsEnd(uint64_t numPixels) {
    return OFF_FB + ((numPixels * 8 + 15) & ~15ull) + 16 + ((numPixels * 4 + 15) & ~15ull) + numPixels * 16;
}
}  // namespace rbuf
